// b2q_sim.cuh — the A1 per-step hot path as SIMT code: one lane per LEG, four lanes per robot, eight robots
// per warp.  Everything a leg needs (its 3 joints, link frames, composite inertias, foot contact rows) lives in
// the lane's registers; the only cross-lane traffic is (a) 4-lane butterfly sums for quantities that meet at the
// floating base and (b) 4-lane broadcasts inside the PGS contact sweep.  `Comm` supplies those two primitives:
// warp shuffles on the GPU (b2q_kernels.cu), a 4-thread barrier exchange in the CPU emulation harness used by the
// CPU-side tests (tests/emu/) — same source, so kernel logic is testable without a GPU.
//
// Reference path replaced (SURVEY.md §8a): Minitaur.Step/ProcessAction/ApplyAction (minitaur.py:248-260,
// 904-947,1384-1401), LaikagoMotorModel.convert_to_torque (laikago_motor.py:103-175), pybullet.stepSimulation
// (minitaur.py:244; Bullet multibody ABA + PGS — restated, see DESIGN.md), ReceiveObservation /
// _GetDelayedObservation (minitaur.py:1151-1193), A1 IK (a1.py:97-110,464-497), ETG layer (rlschool, restated),
// observation packing (EnvWrapper.py:50-109).
//
// Formulation (differs on purpose from the oracle's link-coordinate ABA): all quantities are expressed in the
// base frame B; per leg a 3x3 joint-space block M_k, a 6x3 base coupling F_k and the leg's composite inertia are
// built by the composite-rigid-body method; the four legs only couple through the base, so
//     S = H_base - sum_k F_k M_k^-1 F_k^T   (6x6 Schur complement, = articulated inertia of the base)
// is reduced over the 4 lanes, Cholesky-factored redundantly, and back-substituted per leg.  Contacts are solved
// in contact space: W = J M^-1 J^T (12x12, each lane owns its foot's 3 rows) with projected Gauss-Seidel in
// Bullet's row order (all normals, then all friction rows).
#pragma once
#include "b2q_math.cuh"

namespace b2q {

constexpr int NS = 37;    // state packs per env (21 + 16 action-filter history packs, touched only when the filter is on)
constexpr int NP = 15;    // param packs per env
constexpr int NE = 16;    // ETG packs per env (w[3][20], b[3], pad)
constexpr int OBS_DIM = 49;
constexpr int INFO_DIM = 56;
constexpr int ETG_H = 20;

template <typename T>
struct alignas(4 * sizeof(T)) P4 {
  T x, y, z, w;
};

template <typename T>
struct LegModel {
  T p1[3];       // hip joint origin in the base frame (a1.py:70-73, incl. COM_OFFSET)
  T lhip;        // signed thigh-joint y offset (a1.py:100)
  T com[3][3];   // link COMs in link frames: hip, thigh, calf(+toe)
  T I[3][6];     // inertia about COM, link frame: xx xy xz yy yz zz
  T m[3];
};
template <typename T>
struct Model {
  LegModel<T> leg[4];
  T m0, I0[6];
  T foot_r, l_up, l_low;
  T etg_u[ETG_H][2];
  T base_foot[4][3];
  T etg_mean[12], etg_std[12], etg_istd[12];
  T pose_ori[3];
  T qlo[3], qhi[3];                 // URDF joint limits (a1.py:186-223): hip, upper, lower
  T knee_r;                         // radius of the knee collision sphere at the calf joint (calf / thigh box ends, a1 URDF [EXT])
  // observation layout selected by sensor_mode / normal (EnvWrapper.py:60-109): out[j] = full49[obs_src[j]] * obs_scale[j] + obs_shift[j]
  int obs_dim, obs_identity;
  int obs_src[OBS_DIM];
  T obs_scale[OBS_DIM], obs_shift[OBS_DIM];
};
template <typename T>
struct Cfg {
  T dt; int R; int iters; T erp, warm, margin; int interp; T tau_limit; int settle_steps;
  int filter; T fb0, fb1, fb2, fa1, fa2; int etg; int max_steps;
  T etg_T, etg_T2, etg_sigma_sq, etg_amp, etg_ph0, etg_ph1;
  T w_torso, w_feet, w_up, w_tau, w_stand, w_badfoot, w_footcontact, w_done, reward_p, vel_d;
  int terrain, hf_nx, hf_ny; T hf_x0, hf_y0, hf_cell, hf_icell, idt; const T* hf;
  int clip_cmd; T max_dq;   // A1._ClipMotorCommands (a1.py:440-458)
  int noise_on; T noise[5]; unsigned long long noise_seed;   // Minitaur._AddSensorNoise (minitaur.py:1206-1211)
  int stuck, body_coll;     // stuck termination, non-toe collision count for `badfoot`
  int motor_mode, jlim, extf, knee; T damp[4];   // FEAT variant only: TORQUE mode, joint-limit rows, base push, knee contact rows, Bullet base damping
};
constexpr int STUCK_H = 10;   // control steps of base-position history for the stuck termination
template <typename T>
struct Buffers {
  int N, Dm;
  P4<T>* state;          // [NS][N]
  P4<T>* snap;           // [NS][N] settled snapshot (K2: reset = masked copy)
  P4<T>* snap_obs;       // [12][N]
  const P4<T>* param;    // [NP][N]
  const P4<T>* etg;      // [NE][N]
  P4<T>* ring;           // [Dm][2][12][N]
  int* step_count;       // [N]
  P4<T>* pos_hist;       // [STUCK_H][N] base positions of the last control steps (stuck termination)
  const P4<T>* extf;     // [N] world-frame push on the base (external_force)
};
template <typename T>
struct LaneParam {
  T kp[3], kd[3], iscale[3], mscale[3], m0s, I0s[3], mu, latency;
  V3<T> g;
};
template <typename T>
struct LaneState {
  V3<T> pos; T qx, qy, qz, qw; V3<T> vlin, vang;
  T q[3], qd[3]; T lam_n; int contact;
  T lam_lim[3];   // warm starts of this leg's joint-limit rows (FEAT variant)
};

template <typename T> B2Q_HD void sincos_t(T a, T& s, T& c) { m_sincos(a, s, c); }

// Region clocks of the step kernel, compiled in only with -DB2Q_REGION_CLOCKS (scripts/step_regions.py builds that library apart from
// the product one).  A mark reads clock64(), charges the cycles since the previous mark to the region that ends there and opens the next.
// The product build expands every mark to nothing.
// The part of a substep before the sweep is split in five: PD and kinematics, bias forces and composite inertias, Schur reduction and
// Cholesky (with the unconstrained velocities), contact rows, and the Delassus exchange.
enum { RC_PROLOGUE, RC_PD_KIN, RC_BIAS_INERTIA, RC_SCHUR_CHOL, RC_CONTACT_ROWS, RC_DELASSUS, RC_SWEEP, RC_POST_SWEEP, RC_BETWEEN, RC_EPILOGUE, RC_N };
#if defined(B2Q_REGION_CLOCKS) && defined(__CUDA_ARCH__)
#define B2Q_MARK(cm, region) (cm).mark(region)
#else
#define B2Q_MARK(cm, region) ((void)0)
#endif

// ---------------------------------------------------------------------------------------------------------------
// terrain: plane or bilinear height field
template <typename T>
B2Q_HD T terrain_height(const Cfg<T>& cf, T x, T y, V3<T>& n) {
  if (cf.terrain == 0) { n = mk<T>(0, 0, 1); return T(0); }
  T fx = (x - cf.hf_x0) * cf.hf_icell, fy = (y - cf.hf_y0) * cf.hf_icell;
  fx = m_min(m_max(fx, T(0)), T(cf.hf_nx) - T(1.000001));
  fy = m_min(m_max(fy, T(0)), T(cf.hf_ny) - T(1.000001));
  // In float32 nx - 1.000001 rounds to nx - 1 once nx >= ~17, so the cell index is clamped as an integer too: at or past the far
  // edge the lookup stays in the last cell (tx or ty = 1) and never reads column nx or the row past the end of the field.
  int ix = (int)fx, iy = (int)fy;
  if (ix > cf.hf_nx - 2) ix = cf.hf_nx - 2;
  if (iy > cf.hf_ny - 2) iy = cf.hf_ny - 2;
  T tx = fx - T(ix), ty = fy - T(iy);
  const T* h = cf.hf; int nx = cf.hf_nx;
  T h00 = h[iy * nx + ix], h10 = h[iy * nx + ix + 1], h01 = h[(iy + 1) * nx + ix], h11 = h[(iy + 1) * nx + ix + 1];
  T hh = (1 - tx) * (1 - ty) * h00 + tx * (1 - ty) * h10 + (1 - tx) * ty * h01 + tx * ty * h11;
  T dhdx = ((1 - ty) * (h10 - h00) + ty * (h11 - h01)) * cf.hf_icell;
  T dhdy = ((1 - tx) * (h01 - h00) + tx * (h11 - h10)) * cf.hf_icell;
  T inv = m_rsqrt(dhdx * dhdx + dhdy * dhdy + T(1));
  n = mk<T>(-dhdx * inv, -dhdy * inv, inv);
  return hh;
}

// ---------------------------------------------------------------------------------------------------------------
// closed-form leg kinematics in the base frame (tree-consistent with a1.py:113-129)
template <typename T>
struct LegKin {
  R3<T> R1, R2, R3m;
  V3<T> p1, p2, p3, toe, a2;
};
template <typename T>
B2Q_HD void leg_kin(const Model<T>& md, const LegModel<T>& lm, const T* q, LegKin<T>& K) {
  T s1, c1, s2, c2, s23, c23;
  sincos_t(q[0], s1, c1); sincos_t(q[1], s2, c2); sincos_t(q[1] + q[2], s23, c23);
  K.R1.cx = mk<T>(1, 0, 0); K.R1.cy = mk<T>(0, c1, s1); K.R1.cz = mk<T>(0, -s1, c1);
  K.R2.cx = mk<T>(c2, s1 * s2, -c1 * s2); K.R2.cy = K.R1.cy; K.R2.cz = mk<T>(s2, -s1 * c2, c1 * c2);
  K.R3m.cx = mk<T>(c23, s1 * s23, -c1 * s23); K.R3m.cy = K.R1.cy; K.R3m.cz = mk<T>(s23, -s1 * c23, c1 * c23);
  K.a2 = K.R1.cy;
  K.p1 = mk<T>(lm.p1[0], lm.p1[1], lm.p1[2]);
  K.p2 = K.p1 + K.R1.cy * lm.lhip;
  K.p3 = K.p2 - K.R2.cz * md.l_up;
  K.toe = K.p3 - K.R3m.cz * md.l_low;
}

// closed-form IK, a1.py:97-110 (foot relative to the hip joint origin)
template <typename T>
B2Q_HD void leg_ik(const Model<T>& md, V3<T> f, T lhip, T* ang) {
  T lu = md.l_up, ll = md.l_low;
  T tk = -m_acos((f.x * f.x + f.y * f.y + f.z * f.z - lhip * lhip - ll * ll - lu * lu) / (2 * ll * lu));
  T l = m_sqrt(lu * lu + ll * ll + 2 * lu * ll * m_cos(tk));
  T th = m_asin(-f.x / l) - tk / 2;
  T cc = m_cos(th + tk / 2);
  T c1 = lhip * f.y - l * cc * f.z;
  T s1 = l * cc * f.y + lhip * f.z;
  ang[0] = m_atan2(s1, c1); ang[1] = th; ang[2] = tk;
}

// ETG open-loop reference for this lane's leg: joint offsets relative to pose_ori (SURVEY App. A)
template <typename T, class Comm>
B2Q_HD void etg_act_leg(const Comm& cm, const Cfg<T>& cf, const Model<T>& md, const P4<T>* etg, int N, int env, T t, T* act) {
  const int k = cm.leg();
  if (!cf.etg) { act[0] = act[1] = act[2] = T(0); return; }   // make_env(ETG=0)
  const T two_pi = T(6.283185307179586476925286766559);
  T tt = (k == 0 || k == 3) ? t : t + T(0.5) * cf.etg_T2;
  T om = two_pi / cf.etg_T;
  T x0 = cf.etg_amp * m_sin(cf.etg_ph0 + om * tt), x1 = cf.etg_amp * m_sin(cf.etg_ph1 + om * tt);
  T d[3] = {0, 0, 0};
  const T isig = T(1) / cf.etg_sigma_sq;
  // the env's 63 weights as 16 independent 128-bit loads (all in flight at once), then the 20 RBF features against them
  T e[4 * NE];
#pragma unroll
  for (int p = 0; p < NE; p++) { P4<T> v = ldp(etg, p, N, env); e[4 * p] = v.x; e[4 * p + 1] = v.y; e[4 * p + 2] = v.z; e[4 * p + 3] = v.w; }
#pragma unroll
  for (int h = 0; h < ETG_H; h++) {
    T dx = x0 - md.etg_u[h][0], dy = x1 - md.etg_u[h][1];
    T r = m_exp(-(dx * dx + dy * dy) * isig);
#pragma unroll
    for (int a = 0; a < 3; a++) d[a] += e[a * ETG_H + h] * r;
  }
#pragma unroll
  for (int a = 0; a < 3; a++) d[a] += e[60 + a];
  const LegModel<T>& lm = md.leg[k];
  T ang[3];
  for (int tries = 0; tries < 200; tries++) {  // act_clip: shrink until IK is finite
    V3<T> f = mk<T>(md.base_foot[k][0] + d[0] - lm.p1[0], md.base_foot[k][1] + d[1] - lm.p1[1], md.base_foot[k][2] + d[2] - lm.p1[2]);
    leg_ik(md, f, lm.lhip, ang);
    if (!(m_isnan(ang[0]) || m_isnan(ang[1]) || m_isnan(ang[2]))) break;
    d[0] *= T(0.95); d[1] *= T(0.95); d[2] *= T(0.95);
  }
#pragma unroll
  for (int a = 0; a < 3; a++) act[a] = ang[a] - md.pose_ori[a];
}

// ---------------------------------------------------------------------------------------------------------------
// one physics substep for this lane's leg (+ redundant base)
// General solve of the FEAT variant: 9 rows per leg — toe contact (normal, t1, t2), knee contact (normal, t1, t2: the sphere at the calf
// joint, the first non-toe link a stumbling robot puts down) and one limit row per joint (towards the nearer stop) — = 36 rows, Delassus
// matrix in the robot's shared scratch (cm.scratch(): shared memory on the GPU), projected Gauss-Seidel in Bullet's order: joint-limit
// rows first (non-contact multibody constraints), then the contact normals (toes, knees), then the friction rows — run redundantly by
// the four lanes.  Not the hot path: plain loops, no register-resident matrix.
// Scratch layout: Ya[36][6] | blk[4][45] | vec[36][4] | W[36][36].
constexpr int RPL = 9, NRW = 4 * RPL;
constexpr int SCRATCH_FLOATS = NRW * 6 + 4 * 45 + NRW * 4 + NRW * NRW;
// Parking area of the default body, after its exchange area: per lane the Cholesky factor (21) and reciprocal diagonal (6), the base
// rotation (9), the joint-space contact Jacobian (9) and M_k^-1 (6, symmetric) of the substep, which only the impulse application after
// the sweep reads again.  Stored before the sweep and loaded after it (as are the lane's own Y rows, from the exchange area), they stay
// out of the registers that the sweep's Delassus matrix fills.  Value i of lane k is at SCRATCH_EXCHANGE + 4 i + k: the four lanes of a
// robot use four adjacent banks, and a robot's scratch size is 4 times an odd number (mod 32 banks), so a warp's 32 float accesses hit 32
// different banks.
constexpr int PARK = 51, PARK_L = 0, PARK_LI = 21, PARK_R = 27, PARK_J = 36, PARK_D = 45;
constexpr int SCRATCH_EXCHANGE = 272;   // the default body's exchange area: Y^T [6][12] | vectors [4][12] | active [4] (+pad) | W' [12][12]
constexpr int SCRATCH_FAST = SCRATCH_EXCHANGE + 4 * PARK + 8;
static_assert(SCRATCH_FAST % 32 == 4 || SCRATCH_FAST % 32 == 12 || SCRATCH_FAST % 32 == 20 || SCRATCH_FAST % 32 == 28, "bank spread");
// elements of T in one robot's shared scratch.  Its size and the offsets of its areas are multiples of 4 elements, so the P4<T> loads and
// stores of the exchange stay aligned in both precisions whenever the first robot's scratch is.
B2Q_HD constexpr int scratch_floats(int feat) { return feat ? SCRATCH_FLOATS : SCRATCH_FAST; }
#define JLIM_GAP T(0.06)
template <typename T, class Comm>
B2Q_HD void solve_rows36(const Comm& cm, const Cfg<T>& cf, T mu, const T (*Y)[6] /*[9] rows of this leg*/, const T* u /*[9]*/, const T* blk45 /*leg-local 9x9 block, packed lower*/,
                         const T* targ /*[9]*/, const bool* act /*[9]*/, const T* warm /*[9]*/, T* lk /*[9]*/) {
  const int k = cm.leg();
  T* sh = cm.template scratch<T>();
  T* Ya = sh; T* blk = sh + NRW * 6; T* vec = blk + 4 * 45; T* W = vec + NRW * 4;
  cm.sync();   // the previous substep may have been a fast-path one whose exchange areas overlap this scratch: its loads come first
  for (int e = 0; e < RPL; e++) {
    const int r = RPL * k + e;
    for (int c = 0; c < 6; c++) Ya[r * 6 + c] = Y[e][c];
    vec[r * 4 + 0] = u[e]; vec[r * 4 + 1] = targ[e]; vec[r * 4 + 2] = act[e] ? T(1) : T(0); vec[r * 4 + 3] = warm[e];
  }
  for (int i = 0; i < 45; i++) blk[k * 45 + i] = blk45[i];
  cm.sync();
  // compact list of the ACTIVE rows in the order one iteration visits them (limits, toe normals, knee normals, toe friction, knee
  // friction; legs 0..3 inside each group): typically 6-12 of the 36, so the matrix and the sweep are built on that subset only
  const int grp_row[9] = {6, 7, 8, 0, 3, 1, 2, 4, 5}, grp_par[9] = {-1, -1, -1, -1, -1, 0, 0, 3, 3};
  int idx[NRW], par[NRW], pos_of[NRW], n = 0;
  for (int i = 0; i < NRW; i++) pos_of[i] = -1;
  for (int seg = 0; seg < 5; seg++) {
    const int g0 = seg == 0 ? 0 : seg == 1 ? 3 : seg == 2 ? 4 : seg == 3 ? 5 : 7, g1 = seg == 0 ? 3 : seg == 1 ? 4 : seg == 2 ? 5 : seg == 3 ? 7 : 9;
    for (int f = 0; f < 4; f++)
      for (int g = g0; g < g1; g++) {
        const int r = RPL * f + grp_row[g];
        if (!(vec[r * 4 + 2] > T(0))) continue;
        idx[n] = r; par[n] = grp_par[g] >= 0 ? pos_of[RPL * f + grp_par[g]] : -1; pos_of[r] = n; n++;
      }
  }
  for (int i = 0; i < n; i++) {                       // this lane fills the rows of its own leg
    const int r = idx[i];
    if (r / RPL != k) continue;
    for (int j = 0; j < n; j++) {
      const int c = idx[j];
      T acc = T(0);
      for (int q = 0; q < 6; q++) acc += Ya[r * 6 + q] * Ya[c * 6 + q];
      if (c / RPL == k) { const int a = r - RPL * k, b = c - RPL * k; acc += blk[k * 45 + (a >= b ? a * (a + 1) / 2 + b : b * (b + 1) / 2 + a)]; }
      W[i * NRW + j] = acc;
    }
  }
  cm.sync();
  T lam[NRW], uu[NRW];
  for (int i = 0; i < n; i++) lam[i] = vec[idx[i] * 4 + 3];
  for (int i = 0; i < n; i++) { T a = vec[idx[i] * 4 + 0]; for (int j = 0; j < n; j++) a += W[i * NRW + j] * lam[j]; uu[i] = a; }
  for (int it = 0; it < cf.iters; it++) {
    for (int i = 0; i < n; i++) {
      T ln = lam[i] + (vec[idx[i] * 4 + 1] - uu[i]) / W[i * NRW + i];
      if (par[i] >= 0) { T lim = mu * lam[par[i]]; ln = m_min(m_max(ln, -lim), lim); } else ln = m_max(ln, T(0));
      T dl = ln - lam[i]; lam[i] = ln;
      for (int j = 0; j < n; j++) uu[j] += W[j * NRW + i] * dl;
    }
  }
  for (int e = 0; e < RPL; e++) { const int q = pos_of[RPL * k + e]; lk[e] = q >= 0 ? lam[q] : T(0); }
  cm.sync();                                         // the scratch is reused by the next substep
}

// FEAT = 0: the lean default body (POSITION mode, toe contacts only).  FEAT = 1 adds, behind runtime flags, TORQUE mode, the base
// push, Bullet's base damping and the joint-limit rows; it is a separate instantiation so that the default body stays as
// small as it is (the body is instruction-fetch bound, DESIGN.md §5).
template <typename T, int FEAT, class Comm>
B2Q_HD void substep(const Comm& cm, const Cfg<T>& cf, const Model<T>& md, const LaneParam<T>& pr, LaneState<T>& s,
                    const T* target, T* tau_out, V3<T> fext = V3<T>{0, 0, 0}, const T* hyb = nullptr /*HYBRID: kp[3] | qd*[3] | kd[3] | tau_ff[3]*/) {
  B2Q_MARK(cm, RC_BETWEEN);
  const int k = cm.leg();
  const LegModel<T>& lm = md.leg[k];
  const T dt = cf.dt, idt = cf.idt;
  R3<T> R = quat_to_R(s.qx, s.qy, s.qz, s.qw);
  V3<T> wB = rotT(R, s.vang), vB = rotT(R, s.vlin), gB = rotT(R, pr.g);

  // --- ApplyAction: PD on the current q, qd (pd_latency = 0), laikago_motor.py:165-173
  T tau[3];
#pragma unroll
  for (int j = 0; j < 3; j++) {
    T cmd = target[j];
    if (cf.clip_cmd) cmd = m_min(m_max(cmd, s.q[j] - cf.max_dq), s.q[j] + cf.max_dq);   // a1.py:452-457 (off by default)
    T t = T(-1) * (pr.kp[j] * (s.q[j] - cmd)) - pr.kd[j] * (s.qd[j] - T(0));
    if (FEAT && cf.motor_mode == 1) t = target[j];   // MotorControlMode.TORQUE: the command is the torque (laikago_motor.py:131-134)
    if (FEAT && cf.motor_mode == 2) t = T(-1) * (hyb[j] * (s.q[j] - cmd)) - hyb[6 + j] * (s.qd[j] - hyb[3 + j]) + hyb[9 + j];   // HYBRID: per-command gains, desired velocity, feed-forward torque (laikago_motor.py:152-164)
    if (cf.tau_limit > T(0)) t = m_min(m_max(t, -cf.tau_limit), cf.tau_limit);
    tau[j] = t; tau_out[j] = t;
  }

  // --- kinematics in B
  LegKin<T> K; leg_kin(md, lm, s.q, K);
  const V3<T> a1 = mk<T>(1, 0, 0), a2 = K.a2;
  // the foot's terrain lookup (the substep's one branch before the exchange, on the terrain kind) comes first: the contact rows below then
  // share one basic block with the Schur reduction and the Cholesky chain, and the scheduler can interleave the two independent chains
  V3<T> toe_w = s.pos + rot(R, K.toe), n_w;
  T hgt = terrain_height(cf, toe_w.x, toe_w.y, n_w);
  T dist = toe_w.z - hgt - md.foot_r;
  bool act = dist < cf.margin;
  V3<T> cL[3]; S3<T> IL[3]; T mL[3];
  {
    const R3<T>* Rs[3] = {&K.R1, &K.R2, &K.R3m};
    const V3<T> ps[3] = {K.p1, K.p2, K.p3};
#pragma unroll
    for (int i = 0; i < 3; i++) {
      cL[i] = ps[i] + rot(*Rs[i], mk<T>(lm.com[i][0], lm.com[i][1], lm.com[i][2]));
      S3<T> Il = {lm.I[i][0], lm.I[i][1], lm.I[i][2], lm.I[i][3], lm.I[i][4], lm.I[i][5]};
      S3<T> Ib = rot_sym(*Rs[i], Il);
      T sc = pr.iscale[i];
      IL[i].xx = Ib.xx * sc; IL[i].xy = Ib.xy * sc; IL[i].xz = Ib.xz * sc; IL[i].yy = Ib.yy * sc; IL[i].yz = Ib.yz * sc; IL[i].zz = Ib.zz * sc;
      mL[i] = lm.m[i] * pr.mscale[i];
    }
  }
  B2Q_MARK(cm, RC_PD_KIN);
  // --- velocities and bias accelerations (q'' = 0, base twist derivative = 0, gravity as -g fictitious accel)
  V3<T> w1 = wB + a1 * s.qd[0], w2 = w1 + a2 * s.qd[1], w3 = w2 + a2 * s.qd[2];
  V3<T> pdd0 = cross(wB, vB) - gB;
  V3<T> al1 = cross(wB, a1) * s.qd[0];
  V3<T> pdd1 = pdd0 + cross(wB, cross(wB, K.p1));
  V3<T> al2 = al1 + cross(w1, a2) * s.qd[1];
  V3<T> d21 = K.p2 - K.p1;
  V3<T> pdd2 = pdd1 + cross(al1, d21) + cross(w1, cross(w1, d21));
  V3<T> al3 = al2 + cross(w2, a2) * s.qd[2];
  V3<T> d32 = K.p3 - K.p2;
  V3<T> pdd3 = pdd2 + cross(al2, d32) + cross(w2, cross(w2, d32));
  V3<T> fL[3], nL[3];
  {
    const V3<T> ws[3] = {w1, w2, w3}, als[3] = {al1, al2, al3}, pdds[3] = {pdd1, pdd2, pdd3}, ps[3] = {K.p1, K.p2, K.p3};
#pragma unroll
    for (int i = 0; i < 3; i++) {
      V3<T> r = cL[i] - ps[i];
      V3<T> cdd = pdds[i] + cross(als[i], r) + cross(ws[i], cross(ws[i], r));
      fL[i] = cdd * mL[i];
      nL[i] = mul(IL[i], als[i]) + cross(ws[i], mul(IL[i], ws[i]));
    }
  }
  V3<T> F3 = fL[2], N3 = nL[2] + cross(cL[2] - K.p3, fL[2]);
  V3<T> F2 = fL[1] + F3, N2 = nL[1] + cross(cL[1] - K.p2, fL[1]) + N3 + cross(d32, F3);
  V3<T> F1 = fL[0] + F2, N1 = nL[0] + cross(cL[0] - K.p1, fL[0]) + N2 + cross(d21, F2);
  T hj[3] = {dot(a1, N1), dot(a2, N2), dot(a2, N3)};
  V3<T> NO = N1 + cross(K.p1, F1);  // leg bias wrench about the base origin

  // --- composite inertias about the base origin and the joint-space blocks
  T m3c = mL[2], m2c = mL[1] + m3c, m1c = mL[0] + m2c;
  V3<T> h3c = cL[2] * mL[2], h2c = cL[1] * mL[1] + h3c, h1c = cL[0] * mL[0] + h2c;
  S3<T> I3c = IL[2] + point_inertia(mL[2], cL[2]);
  S3<T> I2c = IL[1] + point_inertia(mL[1], cL[1]) + I3c;
  S3<T> I1c = IL[0] + point_inertia(mL[0], cL[0]) + I2c;
  V3<T> v1 = cross(K.p1, a1), v2 = cross(K.p2, a2), v3 = cross(K.p3, a2);
  V6<T> Fc[3];
  Fc[0].a = mul(I1c, a1) + cross(h1c, v1); Fc[0].l = v1 * m1c + cross(a1, h1c);
  Fc[1].a = mul(I2c, a2) + cross(h2c, v2); Fc[1].l = v2 * m2c + cross(a2, h2c);
  Fc[2].a = mul(I3c, a2) + cross(h3c, v3); Fc[2].l = v3 * m3c + cross(a2, h3c);
  T M11 = dot(a1, Fc[0].a) + dot(v1, Fc[0].l);
  T M21 = dot(a1, Fc[1].a) + dot(v1, Fc[1].l), M22 = dot(a2, Fc[1].a) + dot(v2, Fc[1].l);
  T M31 = dot(a1, Fc[2].a) + dot(v1, Fc[2].l), M32 = dot(a2, Fc[2].a) + dot(v2, Fc[2].l), M33 = dot(a2, Fc[2].a) + dot(v3, Fc[2].l);
  // D = M_k^-1 (symmetric 3x3, cofactors)
  T D[3][3];
  {
    T c00 = M22 * M33 - M32 * M32, c01 = M31 * M32 - M21 * M33, c02 = M21 * M32 - M31 * M22;
    T det = M11 * c00 + M21 * c01 + M31 * c02, id = m_rcp(det);
    D[0][0] = c00 * id; D[0][1] = D[1][0] = c01 * id; D[0][2] = D[2][0] = c02 * id;
    D[1][1] = (M11 * M33 - M31 * M31) * id; D[1][2] = D[2][1] = (M31 * M21 - M11 * M32) * id;
    D[2][2] = (M11 * M22 - M21 * M21) * id;
  }
  T bj[3] = {tau[0] - hj[0], tau[1] - hj[1], tau[2] - hj[2]};
  // F_k (as arrays: Fa[i][c] = component c of column i) and F_k D_k (6x3): FD[j][c] = sum_i F_i[c] D[i][j]
  T Fa[3][6], FD[3][6];
#pragma unroll
  for (int i = 0; i < 3; i++) v6_to_arr(Fc[i], Fa[i]);
#pragma unroll
  for (int j = 0; j < 3; j++) {
#pragma unroll
    for (int c = 0; c < 6; c++) FD[j][c] = m_fma(Fa[2][c], D[2][j], m_fma(Fa[1][c], D[1][j], Fa[0][c] * D[0][j]));
  }

  B2Q_MARK(cm, RC_BIAS_INERTIA);
  // --- leg contribution C_k - (F D) F^T to the base Schur complement and rhs; reduce over the 4 legs (4-lane butterflies)
  T S[21], r6[6];
  {
    // composite C1 as 6x6: [[I1c, hx],[hx^T, m 1]], hx = skew(h1c); lower-left block = hx^T = [[0,hz,-hy],[-hz,0,hx],[hy,-hx,0]]
    const T Z = T(0);
    const T Cf[6][6] = {{I1c.xx, I1c.xy, I1c.xz, Z, -h1c.z, h1c.y},
                        {I1c.xy, I1c.yy, I1c.yz, h1c.z, Z, -h1c.x},
                        {I1c.xz, I1c.yz, I1c.zz, -h1c.y, h1c.x, Z},
                        {Z, h1c.z, -h1c.y, m1c, Z, Z},
                        {-h1c.z, Z, h1c.x, Z, m1c, Z},
                        {h1c.y, -h1c.x, Z, Z, Z, m1c}};
#pragma unroll
    for (int i = 0; i < 6; i++) {
#pragma unroll
      for (int j = 0; j <= i; j++) {
        T v = Cf[i][j];
#pragma unroll
        for (int k = 0; k < 3; k++) v = m_fma(Fa[k][j], -FD[k][i], v);
        S[tri(i, j)] = cm.sum4(v);
      }
    }
    const T NOa[6] = {NO.x, NO.y, NO.z, F1.x, F1.y, F1.z};
#pragma unroll
    for (int i = 0; i < 6; i++) {
      T v = -NOa[i];
#pragma unroll
      for (int k = 0; k < 3; k++) v = m_fma(FD[k][i], -bj[k], v);
      r6[i] = cm.sum4(v);
    }
  }
  {
    // base link: inertia (per-env scaled: I'_ab = sqrt(s_a s_b) I_ab), mass, and its own bias wrench
    T sx = m_sqrt(pr.I0s[0]), sy = m_sqrt(pr.I0s[1]), sz = m_sqrt(pr.I0s[2]);
    S3<T> I0 = {md.I0[0] * sx * sx, md.I0[1] * sx * sy, md.I0[2] * sx * sz, md.I0[3] * sy * sy, md.I0[4] * sy * sz, md.I0[5] * sz * sz};
    T m0 = md.m0 * pr.m0s;
    S[tri(0, 0)] += I0.xx; S[tri(1, 0)] += I0.xy; S[tri(1, 1)] += I0.yy; S[tri(2, 0)] += I0.xz; S[tri(2, 1)] += I0.yz; S[tri(2, 2)] += I0.zz;
    S[tri(3, 3)] += m0; S[tri(4, 4)] += m0; S[tri(5, 5)] += m0;
    V3<T> n0 = cross(wB, mul(I0, wB)), f0 = pdd0 * m0;
    if (FEAT) {
      // Bullet btMultiBody base damping (force = m v (k1 + k2 |v|), torque = I w (k1 + k2 |w|)) and the external push (world frame, at the COM)
      T lv = m_sqrt(dot(vB, vB)), lw = m_sqrt(dot(wB, wB));
      f0 = f0 + vB * (m0 * (cf.damp[0] + cf.damp[1] * lv));
      n0 = n0 + mul(I0, wB) * (cf.damp[2] + cf.damp[3] * lw);
      if (cf.extf) f0 = f0 - rotT(R, fext);
    }
    r6[0] -= n0.x; r6[1] -= n0.y; r6[2] -= n0.z; r6[3] -= f0.x; r6[4] -= f0.y; r6[5] -= f0.z;
  }
  T Li[6];
  chol6(S, Li);      // S now holds L, Li the reciprocal diagonal
  fwd6(S, Li, r6); bwd6(S, Li, r6);  // r6 = base twist derivative (body coordinates)
  V6<T> nud = arr_to_v6(r6);
  T qdd[3];
  {
    T t[3] = {bj[0] - dot6(Fc[0], nud), bj[1] - dot6(Fc[1], nud), bj[2] - dot6(Fc[2], nud)};
#pragma unroll
    for (int j = 0; j < 3; j++) qdd[j] = D[j][0] * t[0] + D[j][1] * t[1] + D[j][2] * t[2];
  }
  // --- unconstrained velocities (body coordinates)
  V3<T> wBs = wB + nud.a * dt, vBs = vB + (nud.l + cross(wB, vB)) * dt;
  T qds[3] = {s.qd[0] + dt * qdd[0], s.qd[1] + dt * qdd[1], s.qd[2] + dt * qdd[2]};

  B2Q_MARK(cm, RC_SCHUR_CHOL);
  // --- contact rows of this lane's foot
  V3<T> t1w = mk<T>(1 - n_w.x * n_w.x, -n_w.x * n_w.y, -n_w.x * n_w.z);
  t1w = t1w * m_rsqrt(dot(t1w, t1w));
  V3<T> t2w = cross(n_w, t1w);
  V3<T> eB[3] = {rotT(R, n_w), rotT(R, t1w), rotT(R, t2w)};
  V3<T> xc = K.toe - eB[0] * md.foot_r;
  T Jk[3][3], u[3], Y[3][6], Wl[3][3];
  {
    V3<T> r1 = cross(a1, xc - K.p1), r2 = cross(a2, xc - K.p2), r3 = cross(a2, xc - K.p3);
#pragma unroll
    for (int e = 0; e < 3; e++) {
      Jk[e][0] = dot(eB[e], r1); Jk[e][1] = dot(eB[e], r2); Jk[e][2] = dot(eB[e], r3);
      V6<T> Jb; Jb.a = cross(xc, eB[e]); Jb.l = eB[e];
      u[e] = dot(Jb.a, wBs) + dot(Jb.l, vBs) + Jk[e][0] * qds[0] + Jk[e][1] * qds[1] + Jk[e][2] * qds[2];
      const T Jba[6] = {Jb.a.x, Jb.a.y, Jb.a.z, Jb.l.x, Jb.l.y, Jb.l.z};
#pragma unroll
      for (int c = 0; c < 6; c++) {
        T g = Jba[c];
#pragma unroll
        for (int j = 0; j < 3; j++) g = m_fma(FD[j][c], -Jk[e][j], g);
        Y[e][c] = g;
      }
      fwd6(S, Li, Y[e]);
    }
#pragma unroll
    for (int e = 0; e < 3; e++) {
      T dj[3];
#pragma unroll
      for (int i = 0; i < 3; i++) dj[i] = D[i][0] * Jk[e][0] + D[i][1] * Jk[e][1] + D[i][2] * Jk[e][2];
#pragma unroll
      for (int e2 = 0; e2 < 3; e2++) Wl[e2][e] = Jk[e2][0] * dj[0] + Jk[e2][1] * dj[1] + Jk[e2][2] * dj[2];
    }
  }
  B2Q_MARK(cm, RC_CONTACT_ROWS);
  T lk[3] = {T(0), T(0), T(0)};   // this lane's own toe impulses
  // extra rows of this leg in the FEAT variant: knee contact (n, t1, t2) and the three joint-limit rows: impulses, base-space Y rows, joint-space Jacobians
  T lkx[6] = {T(0), T(0), T(0), T(0), T(0), T(0)}, Yx[6][6], Jx[6][3];
#pragma unroll
  for (int e = 0; e < 6; e++) {
#pragma unroll
    for (int c = 0; c < 6; c++) Yx[e][c] = T(0);
    Jx[e][0] = Jx[e][1] = Jx[e][2] = T(0);
  }
  bool general = false;
  if constexpr (FEAT != 0) {
    // A limit row can only bind when the joint is within JLIM_GAP of a stop (its target velocity is -gap/dt: 0.06 rad <=> 30 rad/s of
    // approach) and a knee row only when the knee sphere is within the contact margin; other rows are dropped — identically in the
    // oracle — and the general solve runs only for warps in which some robot has such a row (warp-uniform switch: the fast path's
    // shuffles need the whole warp).
    bool need = false;
    T kdist = T(1); V3<T> kn_w = mk<T>(0, 0, 1);
    if (cf.jlim) {
#pragma unroll
      for (int j = 0; j < 3; j++) need = need || (s.q[j] - md.qlo[j] < JLIM_GAP) || (md.qhi[j] - s.q[j] < JLIM_GAP);
    }
    if (cf.knee) {
      V3<T> kw = s.pos + rot(R, K.p3);
      kdist = kw.z - terrain_height(cf, kw.x, kw.y, kn_w) - md.knee_r;
      need = need || (kdist < cf.margin);
    }
    if ((cf.jlim || cf.knee) && cm.any(need)) {
      T Y9[RPL][6], u9[RPL], targ9[RPL], warm9[RPL], blk[45], Jall[RPL][3]; bool act9[RPL];
#pragma unroll
      for (int e = 0; e < 3; e++) {
#pragma unroll
        for (int c = 0; c < 6; c++) Y9[e][c] = Y[e][c];
        u9[e] = u[e]; targ9[e] = T(0); warm9[e] = T(0); act9[e] = act;
        Jall[e][0] = Jk[e][0]; Jall[e][1] = Jk[e][1]; Jall[e][2] = Jk[e][2];
      }
      targ9[0] = dist > T(0) ? -dist * idt : cf.erp * (-dist) * idt; warm9[0] = cf.warm * s.lam_n;
      {
        // knee sphere (calf-joint origin, radius knee_r) against the terrain: the same row construction as the toe's, no warm start
        const bool kact = cf.knee && (kdist < cf.margin);
        V3<T> t1k = mk<T>(1 - kn_w.x * kn_w.x, -kn_w.x * kn_w.y, -kn_w.x * kn_w.z);
        t1k = t1k * m_rsqrt(dot(t1k, t1k));
        V3<T> t2k = cross(kn_w, t1k);
        V3<T> ek[3] = {rotT(R, kn_w), rotT(R, t1k), rotT(R, t2k)};
        V3<T> xk = K.p3 - ek[0] * md.knee_r;
        V3<T> r1 = cross(a1, xk - K.p1), r2 = cross(a2, xk - K.p2), r3 = cross(a2, xk - K.p3);
#pragma unroll
        for (int e = 0; e < 3; e++) {
          T jr[3] = {dot(ek[e], r1), dot(ek[e], r2), dot(ek[e], r3)};
          V6<T> Jb; Jb.a = cross(xk, ek[e]); Jb.l = ek[e];
          u9[3 + e] = dot(Jb.a, wBs) + dot(Jb.l, vBs) + jr[0] * qds[0] + jr[1] * qds[1] + jr[2] * qds[2];
#pragma unroll
          for (int i = 0; i < 6; i++) Yx[e][i] = get6(Jb, i) - (FD[0][i] * jr[0] + FD[1][i] * jr[1] + FD[2][i] * jr[2]);
          fwd6(S, Li, Yx[e]);
          Jx[e][0] = jr[0]; Jx[e][1] = jr[1]; Jx[e][2] = jr[2];
          targ9[3 + e] = T(0); warm9[3 + e] = T(0); act9[3 + e] = kact;
        }
        targ9[3] = kdist > T(0) ? -kdist * idt : cf.erp * (-kdist) * idt;
      }
#pragma unroll
      for (int j = 0; j < 3; j++) {
        // limit row of joint j (a1.py:186-223) towards the nearer stop: Jacobian +-e_j in joint space, none on the base; the same
        // target-velocity rule as a contact (approach up to gap/dt, ERP on violation), Bullet btMultiBodyJointLimitConstraint style
        T glo = s.q[j] - md.qlo[j], ghi = md.qhi[j] - s.q[j], gap = glo, sj = T(1);
        if (ghi < glo) { gap = ghi; sj = T(-1); }
#pragma unroll
        for (int i = 0; i < 6; i++) Yx[3 + j][i] = -sj * FD[j][i];
        fwd6(S, Li, Yx[3 + j]);
        Jx[3 + j][0] = j == 0 ? sj : T(0); Jx[3 + j][1] = j == 1 ? sj : T(0); Jx[3 + j][2] = j == 2 ? sj : T(0);
        u9[6 + j] = sj * qds[j];
        targ9[6 + j] = gap > T(0) ? -gap * idt : cf.erp * (-gap) * idt;
        warm9[6 + j] = cf.warm * s.lam_lim[j];
        act9[6 + j] = cf.jlim && (gap < JLIM_GAP);
      }
#pragma unroll
      for (int e = 0; e < 6; e++) {
#pragma unroll
        for (int c = 0; c < 6; c++) Y9[3 + e][c] = Yx[e][c];
        Jall[3 + e][0] = Jx[e][0]; Jall[3 + e][1] = Jx[e][1]; Jall[3 + e][2] = Jx[e][2];
      }
      // leg-local block J D J^T over the nine rows, packed lower
#pragma unroll
      for (int a = 0; a < RPL; a++) {
        T dj[3];
#pragma unroll
        for (int i = 0; i < 3; i++) dj[i] = D[i][0] * Jall[a][0] + D[i][1] * Jall[a][1] + D[i][2] * Jall[a][2];
#pragma unroll
        for (int b = 0; b <= a; b++) blk[a * (a + 1) / 2 + b] = Jall[b][0] * dj[0] + Jall[b][1] * dj[1] + Jall[b][2] * dj[2];
      }
      T lk9[RPL];
      solve_rows36<T>(cm, cf, pr.mu, Y9, u9, blk, targ9, act9, warm9, lk9);
#pragma unroll
      for (int e = 0; e < 3; e++) lk[e] = lk9[e];
#pragma unroll
      for (int e = 0; e < 6; e++) lkx[e] = lk9[3 + e];
      general = true;
    }
  }
  if (!general) {
  T g[12], Wc[12][12], lam[12];
  // --- the 12x12 contact problem of the robot, built ONCE by its four lanes together and then solved REDUNDANTLY in registers by all
  //     of them (the Gauss-Seidel sweep below has no shuffle on its dependent chain).  Row index r = 3*foot + e (e: 0 normal, 1,2 friction).
  //     Delassus matrix W = J M^-1 J^T: W_ij = Y_i . Y_j (+ the leg-local 3x3 block on the diagonal blocks).  The sweep consumes
  //     W'_ir = W_ir / W_ii (zero diagonal) by source row: Wc[r][i] = W'_ir.
  //     Each lane publishes its foot's three Y rows (transposed, so that the others read them with four-wide vector loads), 1/W_ii, the
  //     unconstrained velocities, target and warm start in the robot's shared scratch; after one exchange it builds the three COLUMNS of W'
  //     that belong to its own source rows (216 multiply-adds, a quarter of the whole matrix's), publishes them, and after the second
  //     exchange every lane loads the whole matrix with four-wide vector loads.  (The substep body is instruction-FETCH bound — DESIGN.md §5
  //     — so instruction count is what matters; the two exchanges replace 120 shuffles.)  Both precisions run this build.
  {
    T* sh = cm.template scratch<T>();
    T* YT = sh;            // [6][12]  YT[c][i] = component c of row i's Y
    T* vecs = sh + 72;     // [4][12]  1/W_ii (0 = inactive row) | unconstrained velocity | target velocity | warm start
    T* afs = sh + 120;     // [4]      foot active
    T* Wp = sh + 128;      // [12][12] Wp[r][i] = W'_ir
    T* park = sh + SCRATCH_EXCHANGE + k;   // park[4 * i]: this lane's value i, read back after the sweep (no other lane touches it)
#pragma unroll
    for (int i = 0; i < 21; i++) park[4 * (PARK_L + i)] = S[i];
#pragma unroll
    for (int i = 0; i < 6; i++) park[4 * (PARK_LI + i)] = Li[i];
    park[4 * (PARK_R + 0)] = R.cx.x; park[4 * (PARK_R + 1)] = R.cx.y; park[4 * (PARK_R + 2)] = R.cx.z; park[4 * (PARK_R + 3)] = R.cy.x; park[4 * (PARK_R + 4)] = R.cy.y;
    park[4 * (PARK_R + 5)] = R.cy.z; park[4 * (PARK_R + 6)] = R.cz.x; park[4 * (PARK_R + 7)] = R.cz.y; park[4 * (PARK_R + 8)] = R.cz.z;
#pragma unroll
    for (int i = 0; i < 9; i++) park[4 * (PARK_J + i)] = Jk[i / 3][i % 3];
    park[4 * (PARK_D + 0)] = D[0][0]; park[4 * (PARK_D + 1)] = D[0][1]; park[4 * (PARK_D + 2)] = D[0][2]; park[4 * (PARK_D + 3)] = D[1][1]; park[4 * (PARK_D + 4)] = D[1][2];
    park[4 * (PARK_D + 5)] = D[2][2];
    const T targ_n = dist > T(0) ? -dist * idt : cf.erp * (-dist) * idt;
    T invo[3];
#pragma unroll
    for (int e = 0; e < 3; e++) {
      T d = Wl[e][e];
#pragma unroll
      for (int c = 0; c < 6; c++) d = m_fma(Y[e][c], Y[e][c], d);
      const T rd = m_rcp(d);   // unconditional, so that the select keeps the exchange in one basic block
      invo[e] = act ? rd : T(0);
      const int i = 3 * k + e;
#pragma unroll
      for (int c = 0; c < 6; c++) YT[c * 12 + i] = Y[e][c];
      vecs[i] = invo[e]; vecs[12 + i] = u[e]; vecs[24 + i] = e == 0 ? targ_n : T(0);
      vecs[36 + i] = (e == 0 && act) ? cf.warm * s.lam_n : T(0);   // warm start of the normal impulse (Bullet 0.85)
    }
    afs[k] = act ? T(1) : T(0);
    cm.sync();
    {
      T Ya[12][6], inv[12];   // Ya[i][c] = component c of row i's Y, inv[i] = 1/W_ii
#pragma unroll
      for (int c = 0; c < 6; c++) {
#pragma unroll
        for (int q = 0; q < 3; q++) {
          const P4<T> v = *reinterpret_cast<const P4<T>*>(YT + c * 12 + 4 * q);
          Ya[4 * q][c] = v.x; Ya[4 * q + 1][c] = v.y; Ya[4 * q + 2][c] = v.z; Ya[4 * q + 3][c] = v.w;
        }
      }
#pragma unroll
      for (int q = 0; q < 3; q++) { const P4<T> v = *reinterpret_cast<const P4<T>*>(vecs + 4 * q); inv[4 * q] = v.x; inv[4 * q + 1] = v.y; inv[4 * q + 2] = v.z; inv[4 * q + 3] = v.w; }
#pragma unroll
      for (int e = 0; e < 3; e++) {          // column r = 3k + e of W': all twelve targets
        const int r = 3 * k + e;
        T col[12];
#pragma unroll
        for (int i = 0; i < 12; i++) {
          T acc = Ya[i][0] * Y[e][0];
#pragma unroll
          for (int c = 1; c < 6; c++) acc = m_fma(Ya[i][c], Y[e][c], acc);
          col[i] = acc * inv[i];
        }
#pragma unroll
        for (int q = 0; q < 3; q++) { P4<T> v; v.x = col[4 * q]; v.y = col[4 * q + 1]; v.z = col[4 * q + 2]; v.w = col[4 * q + 3]; *reinterpret_cast<P4<T>*>(Wp + r * 12 + 4 * q) = v; }
        // the three targets of the lane's own foot also carry the leg-local block (and the zero diagonal): overwrite them
#pragma unroll
        for (int e2 = 0; e2 < 3; e2++) {
          T w = Wl[e2][e];
#pragma unroll
          for (int c = 0; c < 6; c++) w = m_fma(Y[e2][c], Y[e][c], w);
          Wp[r * 12 + 3 * k + e2] = (e2 == e) ? T(0) : w * invo[e2];
        }
      }
    }
    cm.sync();
#pragma unroll
    for (int r = 0; r < 12; r++) {
#pragma unroll
      for (int q = 0; q < 3; q++) { const P4<T> v = *reinterpret_cast<const P4<T>*>(Wp + r * 12 + 4 * q); Wc[r][4 * q] = v.x; Wc[r][4 * q + 1] = v.y; Wc[r][4 * q + 2] = v.z; Wc[r][4 * q + 3] = v.w; }
    }
    // g_i = lam_i + (target_i - u_i) / W_ii is the UNCLAMPED Gauss-Seidel candidate of row i.  A row update
    // lam_j <- clamp(g_j) changes g_i (i != j) by -(W_ij / W_ii) * dlam_j and leaves g_j itself unchanged, so the sweep
    // carries g instead of the contact velocities.  With the warm-started normal impulses lam_3f:
    // g_i = (target_i - u0_i) / W_ii - sum_f W'_{i,3f} lam_3f  (the row's own lam cancels against its W_ii lam term).
    // Inactive feet: zero scale (g frozen at 0), g_n = -BIG => lam stays 0.
    {
      const P4<T> af = *reinterpret_cast<const P4<T>*>(afs);
      const T actf[4] = {af.x, af.y, af.z, af.w};
      T lw[4];
#pragma unroll
      for (int q = 0; q < 3; q++) {
        const P4<T> iv = *reinterpret_cast<const P4<T>*>(vecs + 4 * q), uv = *reinterpret_cast<const P4<T>*>(vecs + 12 + 4 * q);
        const P4<T> tv = *reinterpret_cast<const P4<T>*>(vecs + 24 + 4 * q), lv = *reinterpret_cast<const P4<T>*>(vecs + 36 + 4 * q);
        g[4 * q] = (tv.x - uv.x) * iv.x; g[4 * q + 1] = (tv.y - uv.y) * iv.y; g[4 * q + 2] = (tv.z - uv.z) * iv.z; g[4 * q + 3] = (tv.w - uv.w) * iv.w;
        lam[4 * q] = lv.x; lam[4 * q + 1] = lv.y; lam[4 * q + 2] = lv.z; lam[4 * q + 3] = lv.w;
      }
#pragma unroll
      for (int f = 0; f < 4; f++) lw[f] = lam[3 * f];
#pragma unroll
      for (int i = 0; i < 12; i++) {
#pragma unroll
        for (int f = 0; f < 4; f++) g[i] = m_fma(Wc[3 * f][i], -lw[f], g[i]);
        if (i % 3 == 0 && !(actf[i / 3] > T(0))) g[i] = T(-1e30);
      }
    }
    // third barrier of the substep: every lane's loads of the exchange area are done before any lane's next substep stores into it
    // (measured: alternating between two areas instead costs 10 % — more shared memory per CTA and parity-dependent addressing)
    cm.sync();
  }
  B2Q_MARK(cm, RC_DELASSUS);
  // --- projected Gauss-Seidel, Bullet row order: normals of feet 0..3, then (t1,t2) of feet 0..3.
  //     Row update = clamp -> delta -> 11 independent scalar FFMAs (W'_rr = 0: the row's own candidate is unchanged).
  //     A sweep in which no lambda changes (every dl = 0) leaves g unchanged too, so every later sweep would repeat it exactly: the
  //     lane leaves the loop there and the result is the one all cf.iters sweeps give.  `moved` sums |dl| (zero only if every dl is,
  //     NaN keeps it nonzero); the warp leaves once all 8 robots are at such a fixed point (measured on H100: sweep time -22 %).
  for (int it = 0; it < cf.iters; it++) {
    T moved = T(0);
#pragma unroll
    for (int f = 0; f < 4; f++) {
      const int r = 3 * f;
      T ln = m_max(g[r], T(0));
      T dl = lam[r] - ln; lam[r] = ln;          // dl = -(delta lambda)
      moved += m_abs(dl);
#pragma unroll
      for (int i = 0; i < 12; i++)
        if (i != r) g[i] = m_fma(Wc[r][i], dl, g[i]);
    }
#pragma unroll
    for (int f = 0; f < 4; f++) {
#pragma unroll
      for (int td = 1; td < 3; td++) {
        const int r = 3 * f + td;
        T lim = pr.mu * lam[3 * f];
        T ln = m_min(m_max(g[r], -lim), lim);
        T dl = lam[r] - ln; lam[r] = ln;
        moved += m_abs(dl);
#pragma unroll
        for (int i = 0; i < 12; i++)
          if (i != r) g[i] = m_fma(Wc[r][i], dl, g[i]);
      }
    }
    if (moved == T(0)) break;
  }
  B2Q_MARK(cm, RC_SWEEP);
#pragma unroll
  for (int f = 0; f < 4; f++) if (f == k) { lk[0] = lam[3 * f]; lk[1] = lam[3 * f + 1]; lk[2] = lam[3 * f + 2]; }   // own impulses (no dynamic register indexing)
  {
    // the parked operands of the impulse application (the barrier before the sweep orders these loads after the stores)
    const T* park = cm.template scratch<T>() + SCRATCH_EXCHANGE + k;
#pragma unroll
    for (int i = 0; i < 21; i++) S[i] = park[4 * (PARK_L + i)];
#pragma unroll
    for (int i = 0; i < 6; i++) Li[i] = park[4 * (PARK_LI + i)];
    R.cx = mk<T>(park[4 * (PARK_R + 0)], park[4 * (PARK_R + 1)], park[4 * (PARK_R + 2)]); R.cy = mk<T>(park[4 * (PARK_R + 3)], park[4 * (PARK_R + 4)], park[4 * (PARK_R + 5)]);
    R.cz = mk<T>(park[4 * (PARK_R + 6)], park[4 * (PARK_R + 7)], park[4 * (PARK_R + 8)]);
#pragma unroll
    for (int i = 0; i < 9; i++) Jk[i / 3][i % 3] = park[4 * (PARK_J + i)];
    D[0][0] = park[4 * (PARK_D + 0)]; D[0][1] = D[1][0] = park[4 * (PARK_D + 1)]; D[0][2] = D[2][0] = park[4 * (PARK_D + 2)]; D[1][1] = park[4 * (PARK_D + 3)];
    D[1][2] = D[2][1] = park[4 * (PARK_D + 4)]; D[2][2] = park[4 * (PARK_D + 5)];
    const T* YT = cm.template scratch<T>();   // the lane's own three rows of Y^T, which only this lane writes
#pragma unroll
    for (int e = 0; e < 3; e++) {
#pragma unroll
      for (int c = 0; c < 6; c++) Y[e][c] = YT[c * 12 + 3 * k + e];
    }
  }
  }
  s.lam_n = lk[0]; s.contact = lk[0] > T(0); s.lam_lim[0] = lkx[3]; s.lam_lim[1] = lkx[4]; s.lam_lim[2] = lkx[5];
  // --- apply impulses: sum over feet of Y_f lam_f by a 4-lane butterfly of each lane's own rows (keeps the gathered rows
  //     of the other feet dead after the Delassus matrix is built: 72 fewer live registers across the sweep)
  T z[6];
#pragma unroll
  for (int c = 0; c < 6; c++) z[c] = cm.sum4(Y[0][c] * lk[0] + Y[1][c] * lk[1] + Y[2][c] * lk[2] + (FEAT != 0 ? Yx[0][c] * lkx[0] + Yx[1][c] * lkx[1] + Yx[2][c] * lkx[2] + Yx[3][c] * lkx[3] + Yx[4][c] * lkx[4] + Yx[5][c] * lkx[5] : T(0)));
  bwd6(S, Li, z);
  V6<T> dnu = arr_to_v6(z);
  {
    T jl[3], t[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
      jl[i] = Jk[0][i] * lk[0] + Jk[1][i] * lk[1] + Jk[2][i] * lk[2];
      if (FEAT != 0) jl[i] += Jx[0][i] * lkx[0] + Jx[1][i] * lkx[1] + Jx[2][i] * lkx[2] + Jx[3][i] * lkx[3] + Jx[4][i] * lkx[4] + Jx[5][i] * lkx[5];
      t[i] = jl[i] - dot6(Fc[i], dnu);
    }
#pragma unroll
    for (int j = 0; j < 3; j++) qds[j] += D[j][0] * t[0] + D[j][1] * t[1] + D[j][2] * t[2];
  }
  wBs = wBs + dnu.a; vBs = vBs + dnu.l;
  // --- integrate (semi-implicit Euler; base velocity stored in the world frame as pybullet reports it)
  s.vang = rot(R, wBs); s.vlin = rot(R, vBs);
#pragma unroll
  for (int j = 0; j < 3; j++) { s.qd[j] = qds[j]; s.q[j] += dt * qds[j]; }
  s.pos = s.pos + s.vlin * dt;
  {
    T wx = s.vang.x, wy = s.vang.y, wz = s.vang.z, th = m_sqrt(wx * wx + wy * wy + wz * wz) * dt;
    T sh, cw; sincos_t(T(0.5) * th, sh, cw);
    const T rth = m_rcp(th);   // unconditional (a select, no branch); unused below th = 1e-4
    T kk = th < T(1e-4) ? T(0.5) - th * th * T(1.0 / 48.0) : sh * rth;
    T dx = wx * dt * kk, dy = wy * dt * kk, dz = wz * dt * kk;
    T ox = cw * s.qx + dx * s.qw + dy * s.qz - dz * s.qy;
    T oy = cw * s.qy - dx * s.qz + dy * s.qw + dz * s.qx;
    T oz = cw * s.qz + dx * s.qy - dy * s.qx + dz * s.qw;
    T ow = cw * s.qw - dx * s.qx - dy * s.qy - dz * s.qz;
    T nn = m_rsqrt(ox * ox + oy * oy + oz * oz + ow * ow);
    s.qx = ox * nn; s.qy = oy * nn; s.qz = oz * nn; s.qw = ow * nn;
  }
  B2Q_MARK(cm, RC_POST_SWEEP);
}

// ---------------------------------------------------------------------------------------------------------------
// pack I/O
template <typename T> B2Q_HD P4<T> ldp(const P4<T>* base, int pack, int N, int env) { return base[(size_t)pack * N + env]; }
template <typename T> B2Q_HD void stp(P4<T>* base, int pack, int N, int env, T x, T y, T z, T w) {
  P4<T> p; p.x = x; p.y = y; p.z = z; p.w = w; base[(size_t)pack * N + env] = p;
}

template <typename T, class Comm>
B2Q_HD void load_param(const Comm& cm, const Buffers<T>& B, int env, LaneParam<T>& pr) {
  const int k = cm.leg(), N = B.N;
  P4<T> a = ldp(B.param, 0 + k, N, env), b = ldp(B.param, 4 + k, N, env), c = ldp(B.param, 8 + k, N, env);
  P4<T> d = ldp(B.param, 12, N, env), e = ldp(B.param, 13, N, env), g = ldp(B.param, 14, N, env);
  pr.kp[0] = a.x; pr.kp[1] = a.y; pr.kp[2] = a.z; pr.mu = a.w;
  pr.kd[0] = b.x; pr.kd[1] = b.y; pr.kd[2] = b.z; pr.latency = b.w;
  pr.iscale[0] = c.x; pr.iscale[1] = c.y; pr.iscale[2] = c.z;
  pr.mscale[0] = d.x; pr.mscale[1] = d.y; pr.mscale[2] = d.z; pr.m0s = d.w;
  pr.I0s[0] = e.x; pr.I0s[1] = e.y; pr.I0s[2] = e.z;
  pr.g = mk<T>(g.x, g.y, g.z);
}
template <typename T, class Comm>
B2Q_HD void load_state(const Comm& cm, const P4<T>* st, int N, int env, LaneState<T>& s, T* last_action, T* etg_act, int& has_last, V3<T>& rpy0) {
  const int k = cm.leg();
  P4<T> p0 = ldp(st, 0, N, env), p1 = ldp(st, 1, N, env), p2 = ldp(st, 2, N, env), p3 = ldp(st, 3, N, env);
  P4<T> pq = ldp(st, 4 + k, N, env), pd = ldp(st, 8 + k, N, env), pa = ldp(st, 12 + k, N, env), pe = ldp(st, 16 + k, N, env), pr = ldp(st, 20, N, env);
  s.pos = mk<T>(p0.x, p0.y, p0.z); s.qx = p1.x; s.qy = p1.y; s.qz = p1.z; s.qw = p1.w;
  s.vlin = mk<T>(p2.x, p2.y, p2.z); has_last = p2.w > T(0.5);
  s.vang = mk<T>(p3.x, p3.y, p3.z);
  s.q[0] = pq.x; s.q[1] = pq.y; s.q[2] = pq.z; s.lam_n = pq.w;
  s.qd[0] = pd.x; s.qd[1] = pd.y; s.qd[2] = pd.z; s.contact = pq.w > T(0);   // contact flag = normal impulse > 0 in the last substep
  last_action[0] = pa.x; last_action[1] = pa.y; last_action[2] = pa.z; s.lam_lim[0] = pa.w; s.lam_lim[1] = pe.w; s.lam_lim[2] = pd.w;
  etg_act[0] = pe.x; etg_act[1] = pe.y; etg_act[2] = pe.z;
  rpy0 = mk<T>(pr.x, pr.y, pr.z);
}
template <typename T, class Comm>
B2Q_HD void store_state(const Comm& cm, P4<T>* st, int N, int env, const LaneState<T>& s, const T* last_action, const T* etg_act, int has_last, V3<T> rpy0) {
  const int k = cm.leg();
  if (k == 0) { stp(st, 0, N, env, s.pos.x, s.pos.y, s.pos.z, T(0)); stp(st, 20, N, env, rpy0.x, rpy0.y, rpy0.z, T(0)); }
  if (k == 1) stp(st, 1, N, env, s.qx, s.qy, s.qz, s.qw);
  if (k == 2) stp(st, 2, N, env, s.vlin.x, s.vlin.y, s.vlin.z, T(has_last));
  if (k == 3) stp(st, 3, N, env, s.vang.x, s.vang.y, s.vang.z, T(0));
  stp(st, 4 + k, N, env, s.q[0], s.q[1], s.q[2], s.lam_n);
  stp(st, 8 + k, N, env, s.qd[0], s.qd[1], s.qd[2], s.lam_lim[2]);
  stp(st, 12 + k, N, env, last_action[0], last_action[1], last_action[2], s.lam_lim[0]);
  stp(st, 16 + k, N, env, etg_act[0], etg_act[1], etg_act[2], s.lam_lim[1]);
}
// observation history ring: [Dm][2][12][N]; lane k owns packs 3k..3k+2 = (q, tau0),(qd, tau1),(tau2,-,-,-)
template <typename T>
B2Q_HD void ring_write(const Buffers<T>& B, int slot, int ab, int k, int env, const T* q, const T* qd, const T* tau) {
  P4<T>* base = B.ring + ((size_t)(slot * 2 + ab) * 12) * B.N;
  stp(base, 3 * k + 0, B.N, env, q[0], q[1], q[2], tau[0]);
  stp(base, 3 * k + 1, B.N, env, qd[0], qd[1], qd[2], tau[1]);
  stp(base, 3 * k + 2, B.N, env, tau[2], T(0), T(0), T(0));
}
template <typename T>
B2Q_HD void ring_read(const Buffers<T>& B, int slot, int ab, int k, int env, T* q, T* qd, T* tau) {
  const P4<T>* base = B.ring + ((size_t)(slot * 2 + ab) * 12) * B.N;
  P4<T> a = ldp(base, 3 * k + 0, B.N, env), b = ldp(base, 3 * k + 1, B.N, env), c = ldp(base, 3 * k + 2, B.N, env);
  q[0] = a.x; q[1] = a.y; q[2] = a.z; tau[0] = a.w; qd[0] = b.x; qd[1] = b.y; qd[2] = b.z; tau[1] = b.w; tau[2] = c.x;
}

template <typename T> B2Q_HD T map_pi(T a) {  // MapToMinusPiToPi, minitaur.py:67-83
  const T two_pi = T(6.283185307179586476925286766559), pi = T(3.1415926535897932384626433832795);
  T m = m_fmod(a, two_pi);
  if (m >= pi) m -= two_pi; else if (m < -pi) m += two_pi;
  return m;
}
template <typename T> B2Q_HD T c_prec(T v, T t, T m) { T w = (v - t) * T(2.178272210300875) / m; return m_tanh(w * w); }  // atanh(sqrt(0.95))

// observation row (EnvWrapper.py:60-109 layout; sorted sensor keys, then normalised ETG)
template <typename T, class Comm>
B2Q_HD void write_obs(const Comm& cm, const Model<T>& md, T* obs, bool valid, const LaneState<T>& s, V3<T> start_pos, T dtc, V3<T> rpy0,
                      const T* dq, const T* dqd, const T* etg_act, const T* nz = nullptr /* additive noise on rpy(3), drpy(3) */) {
  if (!valid) return;
  const int k = cm.leg();
  if (k == 0) {
    const T idtc = T(1) / dtc;
    obs[0] = (s.pos.x - start_pos.x) * idtc; obs[1] = (s.pos.y - start_pos.y) * idtc; obs[2] = (s.pos.z - start_pos.z) * idtc;
    V3<T> rpy = quat_to_rpy(s.qx, s.qy, s.qz, s.qw);
    R3<T> R = quat_to_R(s.qx, s.qy, s.qz, s.qw);
    V3<T> wb = rotT(R, s.vang);
    if (nz) { rpy.x += nz[0]; rpy.y += nz[1]; rpy.z += nz[2]; wb.x += nz[3]; wb.y += nz[4]; wb.z += nz[5]; }
    obs[7] = (rpy.x - rpy0.x) * T(10); obs[8] = (rpy.y - rpy0.y) * T(10); obs[9] = (rpy.z - rpy0.z) * T(10);   // /0.1, EnvWrapper.py:87
    obs[10] = wb.x * T(2); obs[11] = wb.y * T(2); obs[12] = wb.z * T(2);                                            // /0.5, EnvWrapper.py:88
  }
  obs[3 + k] = s.contact ? T(1) : T(0);
#pragma unroll
  for (int j = 0; j < 3; j++) {
    obs[13 + 3 * k + j] = (map_pi(dq[j]) - md.pose_ori[j]) * T(10);   // /0.1, EnvWrapper.py:66
    obs[25 + 3 * k + j] = dqd[j];                                          // /1.0, EnvWrapper.py:70
    obs[37 + 3 * k + j] = (etg_act[j] - md.etg_mean[3 * k + j]) * md.etg_istd[3 * k + j];
  }
}

// one output row from a full 49-wide staged row (sensor_mode selection / de-normalisation), element j
template <typename T> B2Q_HD T obs_out_elem(const Model<T>& md, const T* full49, int j) {
  return md.obs_identity ? full49[j] : full49[md.obs_src[j]] * md.obs_scale[j] + md.obs_shift[j];
}

// ---------------------------------------------------------------------------------------------------------------
// reset = masked copy of the settled snapshot (K2); history ring filled with the settled observation
template <typename T, class Comm>
B2Q_HD void reset_lane(const Comm& cm, const Cfg<T>& cf, const Model<T>& md, const Buffers<T>& B, int env, bool valid, T* obs /*49-wide row or null*/,
                       const T* xoff = nullptr /* [N] initial base x offsets (reset(x_noise=)) or null */) {
  const int k = cm.leg(), N = B.N;
  LaneState<T> s; T la[3], ea[3]; int hl; V3<T> rpy0;
  load_state(cm, B.snap, N, env, s, la, ea, hl, rpy0);
  T sq[3], sqd[3], stau[3];
  {
    P4<T> a = ldp(B.snap_obs, 3 * k, N, env), b = ldp(B.snap_obs, 3 * k + 1, N, env), c = ldp(B.snap_obs, 3 * k + 2, N, env);
    sq[0] = a.x; sq[1] = a.y; sq[2] = a.z; stau[0] = a.w; sqd[0] = b.x; sqd[1] = b.y; sqd[2] = b.z; stau[1] = b.w; stau[2] = c.x;
  }
  s.contact = s.lam_n > T(0);
  if (xoff) s.pos.x += xoff[env];
  rpy0 = quat_to_rpy(s.qx, s.qy, s.qz, s.qw);
  etg_act_leg(cm, cf, md, B.etg, N, env, T(0), ea);
  la[0] = la[1] = la[2] = T(0);
  if (valid) {
    store_state(cm, B.state, N, env, s, la, ea, 0, rpy0);
    for (int d = 0; d < B.Dm; d++) { ring_write(B, d, 0, k, env, sq, sqd, stau); ring_write(B, d, 1, k, env, sq, sqd, stau); }
    if (k == 0) B.step_count[env] = 0;
    if (cf.filter) for (int hslot = 0; hslot < 4; hslot++) stp(B.state, 21 + 4 * k + hslot, N, env, sq[0], sq[1], sq[2], T(0));   // init_history(GetMotorAngles()), minitaur.py:1417-1419
  }
  if (obs) write_obs(cm, md, obs, valid, s, s.pos, cf.dt * T(cf.R), rpy0, sq, sqd, ea);
}

// settle: reset pose, hold INIT_MOTOR_ANGLES for settle_steps substeps (a1.py:289-304), then snapshot
template <typename T, int FEAT, class Comm>
B2Q_HD void settle_lane(const Comm& cm, const Cfg<T>& cf, const Model<T>& md, const Buffers<T>& B, int env, bool valid) {
  const int k = cm.leg(), N = B.N;
  LaneParam<T> pr; load_param(cm, B, env, pr);
  LaneState<T> s;
  s.pos = mk<T>(0, 0, T(0.32)); s.qx = s.qy = s.qz = 0; s.qw = 1; s.vlin = mk<T>(0, 0, 0); s.vang = mk<T>(0, 0, 0);
  T tgt[3], tau[3] = {0, 0, 0};
#pragma unroll
  for (int j = 0; j < 3; j++) { s.q[j] = md.pose_ori[j]; s.qd[j] = 0; tgt[j] = md.pose_ori[j]; }
  s.lam_n = 0; s.contact = 0; s.lam_lim[0] = s.lam_lim[1] = s.lam_lim[2] = 0;
  Cfg<T> cs = cf; cs.motor_mode = 0;   // the reset pose is held by the POSITION controller whatever the policy's motor mode (a1.py:289-304)
#pragma unroll 1
  for (int i = 0; i < cf.settle_steps; i++) substep<T, FEAT>(cm, cs, md, pr, s, tgt, tau);
  s.lam_lim[0] = s.lam_lim[1] = s.lam_lim[2] = T(0);   // a reset starts without a joint-limit warm start
  if (valid) {
    T z3[3] = {0, 0, 0};
    store_state(cm, B.snap, N, env, s, z3, z3, 0, mk<T>(0, 0, 0));
    stp(B.snap_obs, 3 * k + 0, N, env, s.q[0], s.q[1], s.q[2], tau[0]);
    stp(B.snap_obs, 3 * k + 1, N, env, s.qd[0], s.qd[1], s.qd[2], tau[1]);
    stp(B.snap_obs, 3 * k + 2, N, env, tau[2], T(0), T(0), T(0));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// one control step (= R physics substeps) for this lane: env.step() of the reference
template <typename T, int FEAT, class Comm>
B2Q_HD void step_lane(const Comm& cm, const Cfg<T>& cf, const Model<T>& md, const Buffers<T>& B, int env, bool valid,
                      const T* action, int donef, int auto_reset, T* obs, T* reward, uint8_t* done, T* info, int obs_env0 = 0, int info_env0 = 0) {
  // `obs` / `info` are row blocks starting at env `obs_env0` / `info_env0`: whole [N][...] arrays (0) or CTA-local staging blocks
  const int k = cm.leg(), N = B.N, R = cf.R;
  const T dtc = cf.dt * T(R);
  LaneParam<T> pr; load_param(cm, B, env, pr);
  LaneState<T> s; T last_action[3], etg_act[3]; int has_last; V3<T> rpy0;
  load_state(cm, B.state, N, env, s, last_action, etg_act, has_last, rpy0);
  int step = B.step_count[env];
  T target[3];
#pragma unroll
  for (int j = 0; j < 3; j++) target[j] = md.pose_ori[j] + etg_act[j] + action[(size_t)env * 12 + 3 * k + j];  // deployment/test.py:95-99
  V3<T> fext = mk<T>(0, 0, 0);
  if (FEAT) {
    if (cf.motor_mode == 1) {   // TORQUE mode: the (already scaled) action is the motor torque, no ETG / pose offset
#pragma unroll
      for (int j = 0; j < 3; j++) target[j] = action[(size_t)env * 12 + 3 * k + j];
    }
    if (cf.extf) { P4<T> f = B.extf[env]; fext = mk<T>(f.x, f.y, f.z); }
  }
  T hyb[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (FEAT && cf.motor_mode == 2) {   // HYBRID: the action is [N][12 motors][q*, kp, qd*, kd, tau_ff] (laikago_motor.py:27-33,152-161), taken as commanded:
#pragma unroll                        // no ETG / pose offset, no interpolation or filtering of the 5-tuples
    for (int j = 0; j < 3; j++) {
      const T* a5 = action + ((size_t)env * 12 + 3 * k + j) * 5;
      target[j] = a5[0]; hyb[j] = a5[1]; hyb[3 + j] = a5[2]; hyb[6 + j] = a5[3]; hyb[9 + j] = a5[4];
    }
  }
  if (cf.filter && !(FEAT && cf.motor_mode == 2)) {  // Minitaur.Step: action = _FilterAction(action) (minitaur.py:250-251); y = b.x_hist - a.y_hist (action_filter.py:111-120)
    P4<T> x1 = ldp(B.state, 21 + 4 * k, N, env), x2 = ldp(B.state, 22 + 4 * k, N, env), y1 = ldp(B.state, 23 + 4 * k, N, env), y2 = ldp(B.state, 24 + 4 * k, N, env);
    T ax1[3] = {x1.x, x1.y, x1.z}, ax2[3] = {x2.x, x2.y, x2.z}, ay1[3] = {y1.x, y1.y, y1.z}, ay2[3] = {y2.x, y2.y, y2.z}, yy[3];
#pragma unroll
    for (int j = 0; j < 3; j++) yy[j] = cf.fb0 * target[j] + cf.fb1 * ax1[j] + cf.fb2 * ax2[j] - cf.fa1 * ay1[j] - cf.fa2 * ay2[j];
    if (valid) {
      stp(B.state, 21 + 4 * k, N, env, target[0], target[1], target[2], T(0)); stp(B.state, 22 + 4 * k, N, env, ax1[0], ax1[1], ax1[2], T(0));
      stp(B.state, 23 + 4 * k, N, env, yy[0], yy[1], yy[2], T(0)); stp(B.state, 24 + 4 * k, N, env, ay1[0], ay1[1], ay1[2], T(0));
    }
#pragma unroll
    for (int j = 0; j < 3; j++) target[j] = yy[j];
  }
  const V3<T> start_pos = s.pos;
  T foot0_x;
  {
    LegKin<T> K; leg_kin(md, md.leg[k], s.q, K);
    R3<T> Rb = quat_to_R(s.qx, s.qy, s.qz, s.qw);
    foot0_x = s.pos.x + rot(Rb, K.toe).x;
  }
  // control-latency bookkeeping (minitaur.py:1172-1193): lags n and n+1 counted from the last substep
  int n_lag = pr.latency > T(0) ? (int)(pr.latency / cf.dt) : 0;
  T alpha = pr.latency > T(0) ? (pr.latency - T(n_lag) * cf.dt) / cf.dt : T(0);
  int max_lag = B.Dm * R - 2; if (n_lag > max_lag) { n_lag = max_lag; alpha = T(0); }
  int ia = ((R - 1 - n_lag) % R + R) % R, ma = (n_lag - (R - 1 - ia)) / R;
  int ib = ((R - 2 - n_lag) % R + R) % R, mb = (n_lag + 1 - (R - 1 - ib)) / R;
  const int slot = step % B.Dm;
  T tau[3] = {0, 0, 0};
  B2Q_MARK(cm, RC_PROLOGUE);
#pragma unroll 1
  for (int i = 0; i < R; i++) {  // Minitaur.Step, minitaur.py:248-260
    T proc[3];
    if (cf.interp && has_last && !(FEAT && cf.motor_mode == 2)) {  // ProcessAction, minitaur.py:1384-1401
      T lerp = T(i + 1) / T(R);
#pragma unroll
      for (int j = 0; j < 3; j++) proc[j] = last_action[j] + lerp * (target[j] - last_action[j]);
    } else {
#pragma unroll
      for (int j = 0; j < 3; j++) proc[j] = target[j];
    }
    substep<T, FEAT>(cm, cf, md, pr, s, proc, tau, fext, hyb);
    if (valid && i == ia) ring_write(B, slot, 0, k, env, s.q, s.qd, tau);
    if (valid && i == ib) ring_write(B, slot, 1, k, env, s.q, s.qd, tau);
  }
  B2Q_MARK(cm, RC_BETWEEN);
#pragma unroll
  for (int j = 0; j < 3; j++) last_action[j] = target[j];
  has_last = 1;
  // delayed (control-latency) observation of this leg's joints
  T dq[3], dqd[3], dtau[3];
  {
    T aq[3], aqd[3], at[3], bq[3], bqd[3], bt[3];
    ring_read(B, ((step - ma) % B.Dm + B.Dm) % B.Dm, 0, k, env, aq, aqd, at);
    ring_read(B, ((step - mb) % B.Dm + B.Dm) % B.Dm, 1, k, env, bq, bqd, bt);
#pragma unroll
    for (int j = 0; j < 3; j++) {
      dq[j] = (T(1) - alpha) * aq[j] + alpha * bq[j];
      dqd[j] = (T(1) - alpha) * aqd[j] + alpha * bqd[j];
      dtau[j] = (T(1) - alpha) * at[j] + alpha * bt[j];
    }
  }
  step += 1;
  T nz6[6] = {0, 0, 0, 0, 0, 0};
  if (cf.noise_on) {   // Minitaur._AddSensorNoise on GetMotorAngles / Velocities / Torques / rpy / rpy rate (minitaur.py:635,762,785,805,880)
    T n4[4];
    philox_normal4<T>(cf.noise_seed, (uint32_t)env, (uint32_t)step, (uint32_t)(16 * k + 0), n4);
#pragma unroll
    for (int j = 0; j < 3; j++) dq[j] += cf.noise[0] * n4[j];
    philox_normal4<T>(cf.noise_seed, (uint32_t)env, (uint32_t)step, (uint32_t)(16 * k + 1), n4);
#pragma unroll
    for (int j = 0; j < 3; j++) dqd[j] += cf.noise[1] * n4[j];
    philox_normal4<T>(cf.noise_seed, (uint32_t)env, (uint32_t)step, (uint32_t)(16 * k + 2), n4);
#pragma unroll
    for (int j = 0; j < 3; j++) dtau[j] += cf.noise[2] * n4[j];
    if (k == 0) {
      philox_normal4<T>(cf.noise_seed, (uint32_t)env, (uint32_t)step, 64u, n4);
      nz6[0] = cf.noise[3] * n4[0]; nz6[1] = cf.noise[3] * n4[1]; nz6[2] = cf.noise[3] * n4[2];
      philox_normal4<T>(cf.noise_seed, (uint32_t)env, (uint32_t)step, 65u, n4);
      nz6[3] = cf.noise[4] * n4[0]; nz6[4] = cf.noise[4] * n4[1]; nz6[5] = cf.noise[4] * n4[2];
    }
  }
  etg_act_leg(cm, cf, md, B.etg, N, env, T(step) * dtc, etg_act);
  T* orow = obs + (size_t)(env - obs_env0) * OBS_DIM;
  write_obs(cm, md, orow, valid, s, start_pos, dtc, rpy0, dq, dqd, etg_act, cf.noise_on ? nz6 : (const T*)nullptr);

  // ---- reward / termination (this repo's definition, DESIGN.md §3)
  R3<T> Rb = quat_to_R(s.qx, s.qy, s.qz, s.qw);
  LegKin<T> K; leg_kin(md, md.leg[k], s.q, K);
  V3<T> toe_w = s.pos + rot(Rb, K.toe), knee_w = s.pos + rot(Rb, K.p3), nrm;
  const T idtc = T(1) / dtc;
  T velx = (s.pos.x - start_pos.x) * idtc;
  T torso = m_min(velx, cf.vel_d);
  T feet = cm.sum4(m_min((toe_w.x - foot0_x) * idtc, cf.vel_d) * T(0.25));
  V3<T> rpy = quat_to_rpy(s.qx, s.qy, s.qz, s.qw);
  T up = T(1) - T(0.5) * (c_prec(rpy.x, T(0), T(0.25)) + c_prec(rpy.y, T(0), T(0.25)));
  T pw = cm.sum4(dtau[0] * dqd[0] + dtau[1] * dqd[1] + dtau[2] * dqd[2]);
  T energy = m_abs(pw) * cf.dt * T(R);  // minitaur.py:810-818
  T kh = terrain_height(cf, knee_w.x, knee_w.y, nrm);
  T badk = (knee_w.z - kh < T(0.03)) ? T(1) : T(0);
  if (cf.body_coll) {
    // non-toe links touching the terrain (what Bullet's contact list on leg links / trunk would report; `badfoot` counts them):
    // knee joint sphere (calf/thigh box end, r 0.02), hip joint (hip cylinder r 0.046, a1 URDF collision shapes [EXT] SURVEY B.3) and
    // this lane's two corners of the trunk box (0.267 x 0.194 x 0.114)
    V3<T> hip_w = s.pos + rot(Rb, K.p2);
    T hh = terrain_height(cf, hip_w.x, hip_w.y, nrm);
    badk = (knee_w.z - kh < T(0.02)) ? T(1) : T(0);
    badk += (hip_w.z - hh < T(0.046)) ? T(1) : T(0);
    const T cx = (k < 2) ? T(0.1335) : T(-0.1335), cy = (k & 1) ? T(0.097) : T(-0.097);
#pragma unroll
    for (int zz = 0; zz < 2; zz++) {
      V3<T> c_w = s.pos + rot(Rb, mk<T>(cx - T(0.012731), cy - T(0.002186), (zz ? T(0.057) : T(-0.057)) - T(0.000515)));
      T ch = terrain_height(cf, c_w.x, c_w.y, nrm);
      badk += (c_w.z - ch < T(0)) ? T(1) : T(0);
    }
  }
  T bad = cm.sum4(badk);
  T nofoot = cm.sum4(s.contact ? T(0) : T(1));
  T meanz = cm.sum4(K.toe.z * T(0.25));
  T above = cm.sum4(K.toe.z > T(0) ? T(1) : T(0));
  bool fin = m_isfinite(s.q[0]) && m_isfinite(s.q[1]) && m_isfinite(s.q[2]) && m_isfinite(s.qd[0]) && m_isfinite(s.qd[1]) && m_isfinite(s.qd[2]) &&
             m_isfinite(s.pos.x) && m_isfinite(s.pos.y) && m_isfinite(s.pos.z) && m_isfinite(s.vlin.x) && m_isfinite(s.vlin.y) && m_isfinite(s.vlin.z);
  T nanf = cm.sum4(fin ? T(0) : T(1));
  bool fall = (Rb.cz.z < T(0.5)) || (meanz > T(-0.1)) || (above > T(0)) || (nanf > T(0));
  T r_torso = cf.w_torso * torso, r_feet = cf.w_feet * feet, r_up = cf.w_up * up, r_tau = -cf.w_tau * energy;
  T r_bad = -cf.w_badfoot * bad, r_fc = -cf.w_footcontact * (nofoot > T(2) ? nofoot - T(2) : T(0)), r_done = fall ? -cf.w_done : T(0);
  T rew = cf.reward_p * (r_torso + r_feet + r_up + r_tau + r_bad + r_fc + r_done);
  T stuckf = T(0);
  if (cf.stuck) {   // rlschool [EXT]: episode ends when the base has not moved over the last STUCK_H control steps (after step 10)
    if (k == 0) {
      if (valid) stp(B.pos_hist, (step - 1) % STUCK_H, N, env, s.pos.x, s.pos.y, s.pos.z, T(0));
      if (step > STUCK_H) {
        T mx = 0, my = 0, mz = 0, vx = 0, vy = 0, vz = 0;
        for (int h = 0; h < STUCK_H; h++) {
          P4<T> ph = ldp(B.pos_hist, h, N, env);
          // relative to the current position (variance is translation invariant; avoids the cancellation of E[x^2]-E[x]^2 far from the origin)
          T dx = ((step - 1) % STUCK_H == h) ? T(0) : ph.x - s.pos.x, dy = ((step - 1) % STUCK_H == h) ? T(0) : ph.y - s.pos.y, dz = ((step - 1) % STUCK_H == h) ? T(0) : ph.z - s.pos.z;
          mx += dx; my += dy; mz += dz; vx += dx * dx; vy += dy * dy; vz += dz * dz;
        }
        const T inv = T(1) / T(STUCK_H);
        mx *= inv; my *= inv; mz *= inv;
        T var = (vx * inv - mx * mx) + (vy * inv - my * my) + (vz * inv - mz * mz);
        stuckf = (var <= T(2e-4) * T(2e-4)) ? T(1) : T(0);
      }
    }
    stuckf = cm.bcast(stuckf, 0);
  }
  bool dn = fall || donef || (cf.max_steps > 0 && step >= cf.max_steps) || (stuckf > T(0));
  if (valid) {
    T* irow = info + (size_t)(env - info_env0) * INFO_DIM;
    if (k == 0) {
      reward[env] = rew; done[env] = dn ? 1 : 0;
      irow[0] = velx; irow[1] = r_torso; irow[2] = r_feet; irow[3] = r_up; irow[4] = r_tau; irow[5] = 0; irow[6] = r_bad; irow[7] = r_fc; irow[8] = r_done;
      irow[9] = nanf > T(0) ? T(1) : T(0); irow[10] = energy; irow[11] = s.pos.z;
      V3<T> wb = rotT(Rb, s.vang);
      irow[36] = rpy.x; irow[37] = rpy.y; irow[38] = rpy.z; irow[39] = wb.x; irow[40] = wb.y; irow[41] = wb.z;
      irow[54] = fall ? T(1) : T(0); irow[55] = T(step);
      B.step_count[env] = step;
    }
#pragma unroll
    for (int j = 0; j < 3; j++) { irow[12 + 3 * k + j] = etg_act[j]; irow[24 + 3 * k + j] = target[j]; irow[42 + 3 * k + j] = s.q[j]; }
    store_state(cm, B.state, N, env, s, last_action, etg_act, has_last, rpy0);
  }
  if (auto_reset) {
    // all four lanes of a robot agree on dn; reset_lane contains exchanges only inside etg/none -> safe to branch per robot
    if (dn) reset_lane(cm, cf, md, B, env, valid, orow);
  }
}

}  // namespace b2q
