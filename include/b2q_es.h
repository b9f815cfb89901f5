/* b2q_es.h — C ABI of the ES population-fitness kernels (K4).  Device pointers, caller's stream, 0 on success.
 *
 * Reference interfaces replaced (QuadrupedalRobots/ETGRL):
 *   b2q_es_accumulate  episode_reward += reward ... until done        train.py:213-249 (run_EStrain_episode)
 *   b2q_es_fitness     fitness_list.append(episode_reward)            train.py:404-413;
 *                      rewards gathered per individual                Dynamic_parallel_model.py:157-167
 * Env e = individual*rollouts + r.  The cross-GPU gather of `fitness` is the caller's NCCL all-gather (SURVEY §8e).
 */
#ifndef B2Q_ES_H
#define B2Q_ES_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
/* per control step: for alive envs ret += reward, len += 1, alive &= !done.  elem_size 4 (float) or 8 (double). */
int b2q_es_accumulate(const void* reward, const uint8_t* done, uint8_t* alive, void* ret, int32_t* len, int n, int elem_size, void* stream);
/* The per-episode statistics of an evaluation (pretrain.py:135-154 run_episode, train.py:202-207 run_evaluate_episodes) in ONE launch per
 * control step.  For every env i that is still alive:
 *   ret[i] += reward[i]; len[i] += 1                                     (bit-identical to b2q_es_accumulate)
 *   term_sum[j*n + i] += info[i*info_dim + cols[j]]     for j < ncols   (per-term episode sums, NaN propagates)
 *   count[i] += info[i*info_dim + count_col] >= thresh                  (when count_col >= 0; NaN does not count)
 *   alive[i] &= !done[i]
 * cols: HOST array of ncols (0..B2Q_ES_MAX_TERMS) info columns, copied by value into the kernel arguments: no device allocation, so the
 * call can be captured in a CUDA graph.  count_col = -1: no count, count may be NULL.  info / term_sum may be NULL when unused.
 * Returns -1 for a NULL required pointer, ncols out of range or a column outside [0, info_dim); -2 on a launch error. */
#define B2Q_ES_MAX_TERMS 16
int b2q_es_accumulate_terms(const void* reward, const uint8_t* done, uint8_t* alive, void* ret, int32_t* len, const void* info, int info_dim,
                            const int32_t* cols, int ncols, void* term_sum, int count_col, double thresh, int32_t* count, int n, int elem_size,
                            void* stream);
/* The per-episode statistics of auto-reset TRAINING envs (train.py:150-157,175,359-366 run_train_episode) in ONE launch per control step,
 * with no host-dependent argument, so the call can be captured in a training iteration's CUDA graph.  Unlike b2q_es_accumulate_terms an
 * episode ends at EVERY done and the next one starts at the following step.  All sums are double, whatever elem_size is.
 *   run [3 + ncols][n] (row r of env i at run[r*n + i]): the running episode: 0 return, 1 length, 2 count, 3 + j term j's sum
 *   win [5 + 2*ncols][n]: the window of closed episodes: 0 episodes, 1 non-finite episodes, 2 Σ return, 3 Σ length, 4 Σ count / length,
 *                         5 + j Σ term j, 5 + ncols + j Σ term j / length
 * For every env i:
 *   run_ret += reward[i]; run_len += 1; run_term[j] += info[i*info_dim + cols[j]]          for j < ncols
 *   run_cnt += (double)info[i*info_dim + count_col] >= thresh                               (when count_col >= 0; NaN does not count)
 *   if done[i]: if run_ret and every run_term[j] are finite, win_episodes += 1 and the episode's sums are added to rows 2..; otherwise
 *               only win_nonfinite += 1.  Then the running row is zeroed.
 * Zero run and win before the first call; zero run to drop the running episodes (after a hard reset), win after reading it.
 * cols: HOST array of ncols (0..B2Q_ES_MAX_TERMS) info columns, passed by value.  count_col = -1: no count (row 4 stays 0).
 * Returns -1 (nothing written) for a NULL required pointer, ncols out of range, a column outside [0, info_dim) or a bad elem_size;
 * -2 on a launch error. */
int b2q_train_episode_stats(const void* reward, const uint8_t* done, const void* info, int info_dim, const int32_t* cols, int ncols, int count_col,
                            double thresh, double* run, double* win, int n, int elem_size, void* stream);
/* fitness[i] = mean over the individual's rollouts of ret; mean_len (may be NULL) likewise for episode lengths. */
int b2q_es_fitness(const void* ret, const int32_t* len, void* fitness, void* mean_len, int pop, int rollouts, int elem_size, void* stream);
/* Batched ETG fit (SURVEY §8f-1): for each individual i, points = prior_points + solutions[i].reshape(6,2) and
 * (w,b) = Opt_with_points(points=points, w0=w0, b0=b0) -- train.py:81-110,405-407 -- in float64 on the device.
 * obs6x20 = ETG_layer.update(t) at ts = [0.5T+0.1, 0, 0.05, 0.1, 0.15, 0.2] (row-major 6x20). w_out [pop,3,20], b_out [pop,3]. */
int b2q_etg_fit(const double* obs6x20, const double* prior_points, const double* solutions, const double* w0, const double* b0, double lamb,
                double precision, double* w_out, double* b_out, int pop, void* stream);
/* Dynamics identification (SURVEY §8f-4): loss_func of model/Dynamic_parallel_model.py:29-41 accumulated on the device.
 * info [n,56] is the step kernel's info output; mean15/std15 = recorded {motor12, drpy3} statistics of THIS control step;
 * acc [n,15] running sums (zero it before an episode); reward[n] = 30 - (max_j mean_t motor_j + max_k mean_t drpy_k)/2.
 * The maxima propagate NaN as the reference's np.max does: a NaN in any one of an env's 15 columns makes its reward NaN, and +inf in
 * one (with no NaN) makes it -inf, so a caller that maps non-finite rewards to a floor (es.DynamicsEvaluator) sees every such env. */
int b2q_dyn_accumulate(const void* info, const void* mean15, const void* std15, void* acc, int n, int elem_size, void* stream);
int b2q_dyn_finish(const void* acc, int steps, void* reward, int n, int elem_size, void* stream);
#ifdef __cplusplus
}
#endif
#endif
