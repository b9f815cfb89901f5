/* b2q_mlp.h — C ABI of the fused 3-layer policy/critic MLP forward (K3) on Hopper tensor cores (wgmma,
 * operands staged in shared memory by bulk async copies).  Device pointers, caller's stream, 0 on success.
 *
 * Reference interfaces replaced (QuadrupedalRobots/ETGRL):
 *   Actor.forward   obs -> relu(l1) -> relu(l2) -> {mean_linear, std_linear}, clamp log_std   model/mujoco_model.py:44-60
 *   Critic.forward  cat(obs,act) -> relu -> relu -> 1   (x2 nets: l1-l3, l4-l6)               model/mujoco_model.py:63-89
 *   SAC.predict     tanh(mean)                                                                  alg/sac.py:60-63
 *   SAC.sample      tanh(mean + exp(log_std)*eps), log_prob with log(1-a^2+1e-6)                alg/sac.py:65-75
 *   MujocoAgent.predict/sample (batch 1 in the reference; batch M here)                         model/mujoco_agent.py:29-41
 * Arithmetic: bf16 operands, f32 accumulation in TMEM, f32 epilogues (bias, ReLU, tanh, clamp, log-prob).
 */
#ifndef B2Q_MLP_H
#define B2Q_MLP_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B2Q_MLP_HIDDEN 256
#define B2Q_MLP_MAX_IN 64
#define B2Q_MLP_MAX_OUT 32
#define B2Q_MLP_PREDICT 0   /* out = tanh(y[:, :A])                                   (actor: out_dim = 2A) */
#define B2Q_MLP_SAMPLE 1    /* out = tanh(mean + exp(clamp(log_std,-20,2)) * eps), logp                    */
#define B2Q_MLP_RAW 2       /* out = y (linear head, e.g. the critic's Q value)                              */

typedef struct B2QMlp* B2QMlpHandle;

/* nets: number of independent weight sets evaluated per launch on the same input (1 actor, 2 twin critics). */
int b2q_mlp_create(int device, int in_dim, int out_dim, int nets, B2QMlpHandle* out);
int b2q_mlp_destroy(B2QMlpHandle h);
const char* b2q_mlp_last_error(B2QMlpHandle h);
/* nn.Linear layouts, float32, device: w1 [256,in_dim], b1 [256], w2 [256,256], b2 [256], w3 [out_dim,256], b3 [out_dim]
 * (for the actor w3 = cat(mean_linear.weight, std_linear.weight)).  Repacks into bf16 UMMA shared-memory images. */
int b2q_mlp_set_weights(B2QMlpHandle h, int net, const float* w1, const float* b1, const float* w2, const float* b2,
                        const float* w3, const float* b3, void* stream);
/* in1 [M,in1_dim] and optional in2 [M,in_dim-in1_dim] are concatenated along the feature axis (critic: obs, action).
 * out [nets,M,A] (PREDICT/SAMPLE: A = out_dim/2; RAW: A = out_dim); logp [M] or NULL (SAMPLE only);
 * raw [nets,M,out_dim] or NULL (pre-activation head, for tests); eps [M,A] or NULL (NULL: counter-based Gaussian from seed). */
int b2q_mlp_forward(B2QMlpHandle h, const float* in1, int in1_dim, const float* in2, int M, int mode, uint64_t seed,
                    const float* eps, float* out, float* logp, float* raw, void* stream);
int64_t b2q_mlp_launch_count(B2QMlpHandle h);

#ifdef __cplusplus
}
#endif
#endif
