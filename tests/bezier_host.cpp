// Host build of the Bezier gait's per-env arithmetic (paddlerobotics_b200/csrc/b2q_bezier.h, the source the device kernel runs), for the
// CPU tests.  Compiled by tests/bezier_host.py with -ffp-contract=off.
#include "../paddlerobotics_b200/csrc/b2q_bezier.h"

using namespace b2q::bezier;

extern "C" {

int bez_state_dim(void) { return BEZ_K; }

// n envs, each from its joint angles q[n][12] through `steps` control steps with the reference foot's contact bits contact[n][steps]:
// tb0[n][12], feet[n][steps][12], ang[n][steps][12], flags[n][steps][3] = (TD, SwRef, StanceSwing) after each step.
void bez_rollout(int n, int steps, const double* q, const unsigned char* contact, double* tb0, double* feet, double* ang, double* flags) {
  for (int e = 0; e < n; e++) {
    double st[BEZ_K];
    reset_env(q + (size_t)e * 12, st);
    for (int j = 0; j < 12; j++) tb0[(size_t)e * 12 + j] = st[S_TB0 + j];
    for (int s = 0; s < steps; s++) {
      const size_t r = (size_t)e * steps + s;
      act_env(st, s + 1, contact[r] != 0, feet + r * 12, ang + r * 12);
      flags[r * 3] = st[S_TD]; flags[r * 3 + 1] = st[S_SWREF]; flags[r * 3 + 2] = st[S_SWING];
    }
  }
}

// the A1 IK of feet [n][4][3] (base frame) -> joint angles [n][12]
void bez_ik(int n, const double* feet, double* ang) {
  for (int e = 0; e < n; e++)
    for (int leg = 0; leg < 4; leg++) foot_ik(leg, feet + (size_t)e * 12 + 3 * leg, ang + (size_t)e * 12 + 3 * leg);
}

}  // extern "C"
