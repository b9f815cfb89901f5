/* b2q_deploy.h — C ABI of the deployment-rehearsal kernels: the control law of the reference's deployment/test.py:93-99 on an env handle,
 * and its optional open-loop Bezier gait (--gait 1).
 *
 * Deployment does not run the in-kernel ETG generator.  Step i of an episode applies
 *     base + act_bound * student(obs) + table[i]                                   (test.py:95-99)
 * and the observation's ETG block is (table[iter] - ETG_mean) / ETG_std, iter = steps since reset   (EnvWrapper.py:103-107).
 * On a handle created with etg_enabled = 0 (the target is pose + action) the two calls below restate that law for every env.  The table
 * row of env e is the handle's own step counter (b2q_get_step_count): 0 after a reset, i + 1 after step i.  No argument changes from one
 * control step to the next, so a whole iteration (obs, policy, act, step) can be captured in a CUDA graph and replayed.
 *
 * Element type of obs, table, action and the record buffers: the handle's (float for precision 0, double for 1).  Device pointers, the
 * caller's stream, 0 on success.  A table row at or past `rows` is never read: that env's ETG block and action become NaN, so the step
 * kernel's non-finite check ends its episode.  B2Q_EINVAL (with b2q_last_error(h) set) for a NULL required pointer or a size out of range.
 */
#ifndef B2Q_DEPLOY_H
#define B2Q_DEPLOY_H
#include <stdint.h>
#include "b2q.h"
#ifdef __cplusplus
extern "C" {
#endif

/* obs [N,obs_dim]: overwrites columns etg_col .. etg_col+11 of every env e with table[r_e] (r_e = the env's step counter), normalised as
 * the step kernel's own ETG block, (table - ETG_mean) * ETG_istd in the handle's type, when `normal` is set, raw otherwise.
 * etg_col = -1: the observation has no ETG block and only the record is written.  Otherwise 0 <= etg_col <= obs_dim - 12.
 * rec_obs [rec_rows,obs_dim] or NULL: env 0's row after the overwrite is copied to rec_obs[r_0] when r_0 < rec_rows
 * (test.py:97 obs_list.append(obs)).  table [rows,12], rows >= 1; obs_dim = b2q_obs_dim(h). */
int b2q_deploy_obs(B2QHandle h, const void* table, int rows, int etg_col, int normal, void* obs, void* rec_obs, int rec_rows, void* stream);

/* action [N,12] = act_bound * policy_out[N,12] (float32, the MLP's output) + table[r_e], in the handle's type with one rounding per
 * operation (no fused multiply-add): the reference's agent.predict(obs) * act_bound + ref_action (test.py:95-96).
 * rec_act [rec_rows,12] or NULL: env 0's action row is copied to rec_act[r_0] when r_0 < rec_rows (test.py:98 action_list, which holds
 * the student plus the table, without the base pose). */
int b2q_deploy_act(B2QHandle h, const float* policy_out, double act_bound, const void* table, int rows, void* action, void* rec_act,
                   int rec_rows, void* stream);

/* Open-loop Bezier gait (test.py --gait 1: GaitWrapper, EnvWrapper.py:123-193, with BezierGait of utilities/Bezier.py and the A1 IK).
 * The gait's joint angles take the place of the base pose: step i applies IK(feet_i) + act_bound * student(obs) + table[i], i.e. on an
 * etg_enabled = 0 handle the action gets IK(feet_i) - POSE_ORI added (POSE_ORI = [0, 0.9, -1.8] x 4).  The gait arithmetic is float64 in
 * both precisions (csrc/b2q_bezier.h).  state: the caller's device buffer [N][B2Q_BEZIER_STATE_DIM] doubles, per env
 *     [0..11] T_b0 (the feet at reset, legs 0..3 x (x, y, z), base frame)  [12] time  [13] TD_time  [14] time_since_last_TD  [15] SwRef
 *     [16] TD (0/1)  [17] StanceSwing of the reference leg (0 stance, 1 swing)
 * Both calls refuse a handle created with etg_enabled = 1. */
#define B2Q_BEZIER_STATE_DIM 18

/* GaitWrapper.reset: T_b0 = the A1 forward kinematics of each env's current joint angles (b2q_get_state columns 13..24); the clock and
 * touchdown state are zeroed and StanceSwing is set to swing, as a fresh BezierGait.  Call it after b2q_reset. */
int b2q_bezier_reset(B2QHandle h, void* state, void* stream);

/* GaitWrapper.step before env.step: with r_e the env's step counter (timesteps = r_e + 1; the first five steps hold the reset feet) and
 * the reference foot's contact bit obs[e][contact_col] == 1 (the FootContactSensor column of the observation the student saw), advances
 * the gait, computes the four feet and their IK and adds (IK - POSE_ORI), rounded once to the handle's type, to action [N,12] in place.
 * An unreachable foot gives NaN angles, so the step kernel's non-finite check ends that env's episode.  0 <= contact_col < obs_dim.
 * rec_feet [rec_rows,4,3] double or NULL: env 0's feet are written to rec_feet[r_0] when r_0 < rec_rows. */
int b2q_bezier_act(B2QHandle h, void* state, int contact_col, const void* obs, void* action, double* rec_feet, int rec_rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif
