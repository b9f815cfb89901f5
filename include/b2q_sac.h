/* b2q_sac.h — C ABI of the SAC learner step (K5/K6): critic + actor losses, backward passes on wgmma tensor cores,
 * Adam, Polyak target sync — all on the device.  Device pointers, caller's stream, 0 on success.
 *
 * Reference interfaces replaced (QuadrupedalRobots/ETGRL):
 *   b2q_sac_learn   SAC.learn = _critic_learn + _actor_learn + sync_target        alg/sac.py:77-118
 *                   (MujocoAgent.learn: model/mujoco_agent.py:43-54; torch.optim.Adam: alg/sac.py:55-58)
 *   b2q_sac_phase   the same in four phases so that a data-parallel learner can all-reduce the gradient buckets
 *                   between gradient computation and the optimiser step (SURVEY §8e collective 2)
 * Parameter vectors are flat float32 [W1|b1|W2|b2|W3|b3] per net (nn.Linear layouts): actor (W3 = cat(mean_linear,
 * std_linear)), then the twin critics [2][...] (l1-l3, l4-l6).  Fixed alpha (no entropy tuning), as the reference.
 */
#ifndef B2Q_SAC_H
#define B2Q_SAC_H
#include <stdint.h>
#include "b2q_mlp.h"
#ifdef __cplusplus
extern "C" {
#endif
typedef struct B2QSac* B2QSacHandle;

/* batch must be a multiple of 128; obs_dim + act_dim <= 64. */
int b2q_sac_create(int device, int obs_dim, int act_dim, int batch, float gamma, float tau, float alpha, float actor_lr, float critic_lr, B2QSacHandle* out);
int b2q_sac_destroy(B2QSacHandle h);
const char* b2q_sac_last_error(B2QSacHandle h);
int b2q_sac_param_count(B2QSacHandle h, int which /*0 actor, 1 twin critic*/);
/* target == NULL copies critic into the target (MujocoAgent.__init__: sync_target(decay=0), mujoco_agent.py:26-27). */
int b2q_sac_set_params(B2QSacHandle h, const float* actor, const float* critic, const float* target, void* stream);
int b2q_sac_get_params(B2QSacHandle h, float* actor, float* critic, float* target, void* stream);
int b2q_sac_get_grads(B2QSacHandle h, float* actor, float* critic, void* stream);
/* obs [B,obs_dim], act [B,act_dim], rew [B], next_obs [B,obs_dim], term [B] (1 - terminal as train.py:148-149);
 * eps_next / eps_cur [B,act_dim]: the N(0,1) draws of the two rsample() calls.  Either may be NULL: that draw then comes from a counter
 * RNG inside the kernels (Philox-4x32-10 keyed by `seed` and the learner's device-side step counter, counter = (row, action)), the backward
 * recomputing exactly the forward's draw — no noise tensors, and a CUDA-graph replay of the call draws fresh noise every step.
 * losses_out: device float[2] = {critic_loss, actor_loss}.
 * b2q_sac_learn == phases 0, 1, 2, 3 of b2q_sac_phase in stream order. */
int b2q_sac_learn(B2QSacHandle h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* term,
                  const float* eps_next, const float* eps_cur, uint64_t seed, float* losses_out, void* stream);
/* phase 0: critic grads (clears the whole gradient bucket first); 1: Adam(critic); 2: actor grads; 3: Adam(actor) + Polyak.
 * The optimiser phases also rewrite the bf16 tensor-core operand images of the nets they update. */
int b2q_sac_phase(B2QSacHandle h, int phase, const float* obs, const float* act, const float* rew, const float* next_obs, const float* term,
                  const float* eps_next, const float* eps_cur, uint64_t seed, void* stream);
/* Behaviour cloning step (BC.BClearn, alg/BC.py:53-72; BCtrain.py:123-138): the student (this handle, obs_dim may be
 * the partial observation obs[3:]) imitates an expert given as two MLP handles evaluated on ref_obs [B,ref_obs_dim].
 * eps [B,act_dim]: the N(0,1) draw of the student's sample().  losses_out device float[2] = {critic_loss, actor_loss}. */
int b2q_sac_bc_learn(B2QSacHandle h, const float* obs, const float* ref_obs, int ref_obs_dim, B2QMlpHandle expert_actor, B2QMlpHandle expert_critic,
                     const float* eps, float* losses_out, void* stream);
/* The same step with an optional eps: NULL draws the student's sample() noise from the counter RNG, Philox-4x32-10 keyed by
 * seed + ctr * 0x9E3779B97F4A7C15 (ctr = the learner's device-side step counter, i.e. the number of completed learn / bc_learn steps),
 * counter = (row, action) — the key rule of b2q_sac_learn's draws.  No noise tensor, and a CUDA-graph replay draws fresh noise every step.
 * b2q_sac_bc_learn(..., eps, ...) == b2q_sac_bc_learn_seeded(..., eps, any seed, ...). */
int b2q_sac_bc_learn_seeded(B2QSacHandle h, const float* obs, const float* ref_obs, int ref_obs_dim, B2QMlpHandle expert_actor,
                            B2QMlpHandle expert_critic, const float* eps_or_null, uint64_t seed, float* losses_out, void* stream);
/* the learner's own forward objects (0 actor, 1 twin critic, 2 target critic): always up to date with the parameters, so a
 * rollout can sample from the policy being trained without copying weights.  Owned by the learner. */
B2QMlpHandle b2q_sac_mlp(B2QSacHandle h, int which);
/* device gradient buckets for an in-place ncclAllReduce: which = 0 actor, 1 twin critic, 2 the ONE flat bucket [actor | critic]
 * (b2q_sac_param_count(h,0) + b2q_sac_param_count(h,1) floats).  With the flat bucket a data-parallel step is
 * phase 0, phase 2, all-reduce, phase 1, phase 3 (both gradients against the pre-update parameters, one collective). */
float* b2q_sac_grad_ptr(B2QSacHandle h, int which);
float* b2q_sac_loss_ptr(B2QSacHandle h);
int64_t b2q_sac_launch_count(B2QSacHandle h);
/* Learner snapshot: a header (magic, version, sizes, obs_dim, act_dim, batch, gamma, tau, alpha, both learning rates), then the actor,
 * critic and target parameters, the four Adam moment buffers, the loss buffer and the device step counter with the closing-Adam ticket.
 * dst / src: DEVICE pointers of b2q_sac_snapshot_bytes(h) bytes, 16-byte aligned.  Save is stream-ordered with no host sync.  Load
 * reads the header to the host (waited for), returns B2Q_EINVAL for a blob of another shape, hyper-parameter set, format or size
 * (b2q_sac_last_error names the field), then copies the buffers and rebuilds the bf16 tensor-core operand images with the packer
 * of b2q_sac_set_params, so the next learn is bit-identical to the saved learner's. */
int64_t b2q_sac_snapshot_bytes(B2QSacHandle h);
/* Byte offset in the snapshot of the loss buffer (4 floats: this learner's last losses, the one part that data-parallel ranks do not
 * share); -1 for a NULL handle. */
int64_t b2q_sac_snapshot_loss_offset(B2QSacHandle h);
int b2q_sac_snapshot_save(B2QSacHandle h, void* dst, void* stream);
int b2q_sac_snapshot_load(B2QSacHandle h, const void* src, void* stream);
#ifdef __cplusplus
}
#endif
#endif
