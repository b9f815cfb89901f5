// b2q_bezier.h — per-env arithmetic of the reference's open-loop Bezier gait (deployment --gait 1): GaitWrapper
// (deployment/envs/EnvWrapper.py:123-193) driving BezierGait.GenerateTrajectoryX (deployment/utilities/Bezier.py:530-612) with the
// parameters of BezierStepper (deployment/utilities/SpotOL.py:23-258) and the A1 leg kinematics (deployment/robots/a1.py:97-173,464-490).
// Plain float64 arithmetic, __host__ __device__: b2q_deploy.cu runs it one thread per env, and tests/bezier_host.cpp compiles the same
// source for the CPU so the tests can hold it against the reference's own trajectories (tests/golden/bezier_gait.npz).
//
// State of one env: BEZ_K doubles (the caller's [N][BEZ_K] buffer, include/b2q_deploy.h)
//   [0..11]  T_b0: the feet in the base frame at reset, legs 0..3 x (x, y, z)  (GaitWrapper.reset, EnvWrapper.py:145-151)
//   [12] time  [13] TD_time  [14] time_since_last_TD  [15] SwRef  [16] TD (0/1)  [17] StanceSwing of the reference leg (0 stance, 1 swing)
// Constant parameters (GaitWrapper.step, EnvWrapper.py:158-175): StateMachine() in its default FWD mode only clips and returns the
// constructor's values (SpotOL.py:111-183): StepLength 0.04, LateralFraction 0, YawRate 0, StepVelocity = the wrapper's 0.5,
// PenetrationDepth 0.003; ClearanceHeight is forced to 0.05.  All lie inside their clip limits.  For the first five steps
// (`timesteps > 5` after the increment) the wrapper calls GenerateTrajectoryX(0, 0, 0, 1, ...) instead, which holds the reset feet.
//
// With LateralFraction = YawRate = 0 the lateral and rotational terms of SwingStep / StanceStep (Bezier.py:337-411) are sums of signed
// zeros, which leave the feet's x and y unchanged, with one exception kept here: the rotational BezierSwing(phase, YawRate dt, phi_arc,
// clearance) still has the clearance profile in z, so the swing height is twice the Bezier z curve.  YawCircle's phi_arc (and the
// Prev_fxyz it reads) only multiplies those zeros, so it is not computed.  The reference's Phases list aliases dSref, and dSref's default
// list is shared between BezierGait instances (Bezier.py:23-26,54,437); neither changes the output, because each leg's lag is written
// just before it is read (:592-600), so each leg's lag here is a constant.
#pragma once
#include "b2q_math.cuh"

namespace b2q {
namespace bezier {

constexpr int BEZ_K = 18;
enum { S_TB0 = 0, S_TIME = 12, S_TD_TIME = 13, S_TSL = 14, S_SWREF = 15, S_TD = 16, S_SWING = 17 };

constexpr double DT = 0.026;          // BezierGait(dt=self.dt): the control step (test.py --dt)
constexpr double TSWING = 0.2;        // BezierGait's Tswing default (Bezier.py:23)
constexpr double L_UP = 0.2, L_LOW = 0.2, L_HIP = 0.08505;   // a1.py:98-100

// HIP_OFFSETS = the hip positions + COM_OFFSET (a1.py:70-73), A1 leg order 0..3
B2Q_HD double hip_offset(int leg, int c) {
  const double com[3] = {-0.012731, -0.002186, -0.000515};
  const double hip[3] = {(leg < 2) ? 0.183 : -0.183, (leg & 1) ? 0.047 : -0.047, 0.0};
  return hip[c] + com[c];
}
// INIT_MOTOR_ANGLES (a1.py:83) = POSE_ORI: the base pose an etg_enabled = 0 handle adds to its action, joint j of a leg
B2Q_HD double pose_ori(int j) { return j == 0 ? 0.0 : j == 1 ? 0.9 : -1.8; }
B2Q_HD double hip_sign(int leg) { return (leg & 1) ? 1.0 : -1.0; }   // (-1)**(leg_id + 1), a1.py:172,487

// foot_position_in_hip_frame (a1.py:113-129) + HIP_OFFSETS (foot_positions_in_base_frame, :167-173)
B2Q_HD void foot_fk(int leg, const double* ang, double* p) {
  const double lh = L_HIP * hip_sign(leg);
  const double ld = m_sqrt(L_UP * L_UP + L_LOW * L_LOW + 2 * L_UP * L_LOW * m_cos(ang[2]));
  const double eff = ang[1] + ang[2] / 2;
  const double off_z = -ld * m_cos(eff);
  p[0] = -ld * m_sin(eff) + hip_offset(leg, 0);
  p[1] = (m_cos(ang[0]) * lh - m_sin(ang[0]) * off_z) + hip_offset(leg, 1);
  p[2] = (m_sin(ang[0]) * lh + m_cos(ang[0]) * off_z) + hip_offset(leg, 2);
}

// ComputeMotorAnglesFromFootLocalPosition (a1.py:464-497, zero motor offsets, unit directions) = foot_position_in_hip_frame_to_joint_angle
// (a1.py:97-110) of the foot relative to the hip.  No shrink-until-finite loop: an unreachable foot gives NaN angles, as in the reference.
B2Q_HD void foot_ik(int leg, const double* foot, double* ang) {
  const double lh = L_HIP * hip_sign(leg);
  const double x = foot[0] - hip_offset(leg, 0), y = foot[1] - hip_offset(leg, 1), z = foot[2] - hip_offset(leg, 2);
  const double tk = -m_acos((x * x + y * y + z * z - lh * lh - L_LOW * L_LOW - L_UP * L_UP) / (2 * L_LOW * L_UP));
  const double l = m_sqrt(L_UP * L_UP + L_LOW * L_LOW + 2 * L_UP * L_LOW * m_cos(tk));
  const double th = m_asin(-x / l) - tk / 2;
  const double cc = m_cos(th + tk / 2);
  const double c1 = lh * y - l * cc * z;
  const double s1 = l * cc * y + lh * z;
  ang[0] = m_atan2(s1, c1); ang[1] = th; ang[2] = tk;
}

// GaitWrapper.reset (EnvWrapper.py:140-153): T_b0 from the joint angles q[12], and a fresh BezierGait (Bezier.py:22-54): clock and
// touchdown state zero, StanceSwing = SWING.
B2Q_HD void reset_env(const double* q, double* st) {
  for (int leg = 0; leg < 4; leg++) foot_fk(leg, q + 3 * leg, st + S_TB0 + 3 * leg);
  st[S_TIME] = st[S_TD_TIME] = st[S_TSL] = st[S_SWREF] = st[S_TD] = 0.0;
  st[S_SWING] = 1.0;
}

// BernSteinPoly sums of BezierSwing (Bezier.py:186-277) at LateralFraction 0: the forward (x) and vertical (z) profiles for half step
// length L, each term point * C(11, k) * t^k * (1 - t)^(11 - k), summed from k = 0.
B2Q_HD void bezier_swing(double t, double L, double clearance, double& sx, double& sz) {
  const double binom[12] = {1, 11, 55, 165, 330, 462, 462, 330, 165, 55, 11, 1};
  const double X[12] = {-L, -L * 1.4, -L * 1.5, -L * 1.5, -L * 1.5, 0.0, 0.0, 0.0, L * 1.5, L * 1.5, L * 1.4, L};
  const double c9 = clearance * 0.9, c11 = clearance * 1.1;
  const double Z[12] = {0.0, 0.0, c9, c9, c9, c9, c9, c11, c11, c11, 0.0, 0.0};
  sx = 0.0; sz = 0.0;
  for (int k = 0; k < 12; k++) {
    const double tk = pow(t, (double)k), uk = pow(1 - t, (double)(11 - k));
    sx += X[k] * binom[k] * tk * uk;
    sz += Z[k] * binom[k] * tk * uk;
  }
}

// One GaitWrapper.step (EnvWrapper.py:155-190) for one env: `timesteps` is the wrapper's counter after its increment (control steps since
// reset + 1), `contact0` the reference foot's FootContactSensor bit.  Advances the state and writes the four feet [12] (base frame) and
// their IK joint angles [12].
B2Q_HD void act_env(double* st, int timesteps, bool contact0, double* feet, double* ang) {
  double L = 0.04, vel = 0.5;
  if (!(timesteps > 5)) { L = 0.0; vel = 1.0; }                  // EnvWrapper.py:177-183
  const double clearance = 0.05, pd = 0.003;
  double time = st[S_TIME], td_time = st[S_TD_TIME], tsl = st[S_TSL], swref = st[S_SWREF];
  bool td = st[S_TD] != 0.0;
  double swing = st[S_SWING];
  // GenerateTrajectoryX, Bezier.py:555-587 (vel is never 0 here, so the vel == 0 branch of :557-562 is left out)
  double Tstance = 2.0 * m_abs(L) / m_abs(vel);
  if (Tstance < DT) { Tstance = 0.0; L = 0.0; td = false; time = 0.0; tsl = 0.0; }
  else if (Tstance > 1.3 * TSWING) Tstance = 1.3 * TSWING;
  if (contact0 && Tstance > DT) td = true;
  // Increment with CheckTouchDown, Bezier.py:149-184
  const double Tstride = Tstance + TSWING;
  if (swref >= 0.9 && td) { td_time = time; td = false; swref = 0.0; }
  tsl = time - td_time;
  if (tsl > Tstride) tsl = Tstride;
  else if (tsl < 0.0) tsl = 0.0;
  time += DT;
  if (Tstride < TSWING + DT) { time = 0.0; tsl = 0.0; td_time = 0.0; swref = 0.0; }
  for (int leg = 0; leg < 4; leg++) {
    const double* p = st + S_TB0 + 3 * leg;
    double dx = 0.0, dz = 0.0;
    if (Tstance > 0.0) {
      // GetPhase with Get_ti (Bezier.py:75-147); lags FL, FR, BL, BR = 0, 0.5, 0.5, 0 (:592-600), the reference leg is index 0
      const double lag = (leg == 1 || leg == 2) ? 0.5 : 0.0;
      double ti = tsl - lag * Tstride;
      if (ti < -TSWING) ti += Tstride;
      bool sw = false;
      double phase = 0.0;
      if (ti >= 0.0 && ti <= Tstance) {
        phase = ti / Tstance;
        if (leg == 0) swing = 0.0;
      } else {
        if (ti >= -TSWING && ti < 0.0) { sw = true; phase = (ti + TSWING) / TSWING; }
        else if (ti > Tstance && ti <= Tstride) { sw = true; phase = (ti - Tstance) / TSWING; }
        if (phase >= 1.0) phase = 1.0;                      // otherwise (ti past the stride) the leg takes the stance branch at phase 0
        if (leg == 0) {
          swing = sw ? 1.0 : 0.0;
          swref = phase;
          if (swref >= 0.999) td = true;
        }
      }
      if (sw) {                                             // SwingStep: the forward and the rotational BezierSwing (Bezier.py:337-373)
        double sz;
        bezier_swing(phase, L, clearance, dx, sz);
        dz = sz + sz;
      } else {                                              // StanceStep: SineStance (Bezier.py:279-300,375-411); L != 0 here
        dx = L * (1.0 - 2.0 * phase);
        dz = -pd * m_cos((3.141592653589793 * dx) / (2.0 * L));
      }
    }
    double* f = feet + 3 * leg;
    f[0] = p[0] + dx; f[1] = p[1]; f[2] = p[2] + dz;       // Bezier.py:609-611
    foot_ik(leg, f, ang + 3 * leg);
  }
  st[S_TIME] = time; st[S_TD_TIME] = td_time; st[S_TSL] = tsl; st[S_SWREF] = swref; st[S_TD] = td ? 1.0 : 0.0; st[S_SWING] = swing;
}

}  // namespace bezier
}  // namespace b2q
