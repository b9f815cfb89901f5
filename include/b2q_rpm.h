/* b2q_rpm.h — device-resident replay memory (SURVEY §8f-2): the ring storage lives in caller-owned device tensors,
 * these two kernels append a whole batch of env transitions per control step and gather a uniformly sampled minibatch,
 * so the SAC loop has no host traffic.  Replaces parl.utils.ReplayMemory.append / sample_batch as used at
 * ETGRL/train.py:159,164 (and BCreplay_buffer.py:21-84).  float32 storage.  0 on success. */
#ifndef B2Q_RPM_H
#define B2Q_RPM_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
/* writes n rows at ring positions (pos + i) % capacity.  valid_or_null is ignored: every row is written.  The masked append is
 * b2q_rpm_append_masked_cursor below. */
int b2q_rpm_append(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term,
                   const float* obs, const float* act, const float* rew, const float* next_obs, const float* term, const uint8_t* valid_or_null,
                   int n, int obs_dim, int act_dim, int pos, int capacity, void* stream);
/* gathers `batch` rows with indices drawn uniformly in [0,size) from a counter RNG keyed by seed. */
int b2q_rpm_sample(const float* s_obs, const float* s_act, const float* s_rew, const float* s_next, const float* s_term,
                   float* obs, float* act, float* rew, float* next_obs, float* term, int batch, int obs_dim, int act_dim, int size,
                   uint64_t seed, void* stream);
/* The same two operations with a DEVICE-side cursor: state = device int64[3] {ring position, fill level, sample counter}.  append writes at
 * (state[0] + i) % capacity and then advances position and fill level; sample draws from [0, state[1]) with the key seed + state[2] and then
 * increments the counter.  Nothing about the ring's progress is a kernel argument, so a whole training iteration (policy forward, env step,
 * append, sample, learn) can be captured ONCE in a CUDA graph and replayed.  The fill level must be >= 1 when sample runs. */
int b2q_rpm_append_cursor(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term,
                          const float* obs, const float* act, const float* rew, const float* next_obs, const float* term,
                          int n, int obs_dim, int act_dim, int capacity, long long* state, void* stream);
int b2q_rpm_sample_cursor(const float* s_obs, const float* s_act, const float* s_rew, const float* s_next, const float* s_term,
                          float* obs, float* act, float* rew, float* next_obs, float* term, int batch, int obs_dim, int act_dim,
                          uint64_t seed, long long* state, void* stream);
/* Masked append on the device cursor: writes exactly the rows with valid[i] != 0 (one byte per row), in ascending i, at
 * (state[0] + rank_i) % capacity, rank_i = the number of valid rows before i; then advances position and fill level by the number of
 * valid rows (the sample counter is unchanged).  That number stays on the device: no kernel argument depends on it and nothing
 * synchronises, so a captured call replays correctly when the mask contents change.  1 <= n <= capacity; an all-zero mask changes
 * nothing.  Two launches, deterministic. */
int b2q_rpm_append_masked_cursor(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term,
                                 const float* obs, const float* act, const float* rew, const float* next_obs, const float* term,
                                 const uint8_t* valid, int n, int obs_dim, int act_dim, int capacity, long long* state, void* stream);

/* ---- behaviour cloning (BCtrain.py:53-59,77-84,120; BCreplay_buffer.py:21-84): a ring of (student row, expert row) pairs.
 *
 * b2q_bc_observe: one launch per control step.  obs [n, obs_dim] (the expert's view, obs_dim >= 37) ->
 *   student [n, obs_dim - 3] = obs[:, 3:] + sensor noise, the noise of BCtrain.py:55-58 on expert columns 7:10, 10:13, 13:25, 25:37 with
 *   sigma 0.6, 0.2, 0.1, 0.5 (the reference's sigmas divided by the sensor normalisers) and on no other column.  The value of a noisy
 *   column c of row i is the float32 sum  obs[i, c] + (float)(sigma * z), both operations rounded separately (no fused multiply-add), where
 *     z = Philox-4x32-10 / Box-Muller normal of b2q_philox.cuh with the 64-bit key  (uint64)seed | (uint64)step << 32
 *         (key word 0 = seed, key word 1 = step) and the counter (i, c, 0x9E3779B9, 0): env row i, EXPERT column c.
 *   noise == 0: the student row is an exact copy of obs[i, 3:].
 *   ring_obs [capacity, obs_dim - 3] / ring_ref [capacity, obs_dim] (both or neither): when given, the pair (student row, obs row) is also
 *   written at slot (pos + i) % capacity, as b2q_rpm_append does (1 <= n <= capacity, 0 <= pos).  NULL ring: the student rows only.
 *
 * b2q_bc_gather_cursor: off = state[0] (device int64); row r of the batch is ring row perm[off + r] (perm: device int64, entries in
 *   [0, capacity)): out_obs [batch, obs_dim] = ring_obs[perm[off + r]], out_ref [batch, ref_dim] = ring_ref[perm[off + r]], copied
 *   bit for bit; then state[0] += batch (a second, one-thread launch).  Rows with off + r >= perm_len are not written.  No argument depends
 *   on the position within the pass, so a CUDA graph of G (gather, update) steps replays over consecutive windows. */
int b2q_bc_observe(const float* obs, int n, int obs_dim, float* student, float* ring_obs, float* ring_ref, int pos, int capacity,
                   uint32_t seed, uint32_t step, int noise, void* stream);
int b2q_bc_gather_cursor(const float* ring_obs, const float* ring_ref, const int64_t* perm, int perm_len, long long* state,
                         float* out_obs, float* out_ref, int batch, int obs_dim, int ref_dim, void* stream);
#ifdef __cplusplus
}
#endif
#endif
