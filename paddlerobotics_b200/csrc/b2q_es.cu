// b2q_es.cu — K4: ES population fitness on device (include/b2q_es.h).
// Replaces `fitness_list.append(episode_reward)` (train.py:404-413) and the per-actor reward gather of
// Dynamic_parallel_model.py:152-167: per-env episode return / length accumulation with first-done freezing, then a
// segmented mean over each individual's rollouts.  The all-gather across GPUs is done by the caller (NCCL).
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/b2q_es.h"

namespace {

template <typename T>
__global__ void es_accumulate_kernel(const T* __restrict__ reward, const uint8_t* __restrict__ done, uint8_t* __restrict__ alive,
                                     T* __restrict__ ret, int32_t* __restrict__ len, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (alive[i]) {               // run_EStrain_episode: accumulate until the env reports done (train.py:221-246)
    ret[i] += reward[i];
    len[i] += 1;
    if (done[i]) alive[i] = 0;
  }
}

struct TermCols { int32_t c[B2Q_ES_MAX_TERMS]; };   // by value in the kernel's parameter space

// es_accumulate_kernel plus the per-term sums and the success count of the same alive envs (include/b2q_es.h).  The loop over the
// columns is unrolled to B2Q_ES_MAX_TERMS so that every cols.c[j] is a constant-bank read, never a local copy of the struct.
template <typename T>
__global__ void es_accumulate_terms_kernel(const T* __restrict__ reward, const uint8_t* __restrict__ done, uint8_t* __restrict__ alive,
                                           T* __restrict__ ret, int32_t* __restrict__ len, const T* __restrict__ info, int info_dim,
                                           TermCols cols, int ncols, T* __restrict__ term_sum, int count_col, T thresh,
                                           int32_t* __restrict__ count, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !alive[i]) return;
  ret[i] += reward[i];
  len[i] += 1;
  const T* row = info + (size_t)i * info_dim;
#pragma unroll
  for (int j = 0; j < B2Q_ES_MAX_TERMS; j++)
    if (j < ncols) term_sum[(size_t)j * n + i] += row[cols.c[j]];
  if (count_col >= 0) count[i] += row[count_col] >= thresh ? 1 : 0;   // NaN >= thresh is false
  if (done[i]) alive[i] = 0;
}

// Per-episode statistics of auto-reset training envs (include/b2q_es.h, b2q_train_episode_stats).  Sums in double whatever T is; an
// episode is closed at every done.  Term sums stay in registers between the running update and the fold, so each row is read once.
template <typename T>
__global__ void train_episode_stats_kernel(const T* __restrict__ reward, const uint8_t* __restrict__ done, const T* __restrict__ info, int info_dim,
                                           TermCols cols, int ncols, int count_col, double thresh, double* __restrict__ run,
                                           double* __restrict__ win, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t N = (size_t)n;
  const T* row = info + (size_t)i * info_dim;
  double ret = run[i] + (double)reward[i];
  double len = run[N + i] + 1.0;
  double cnt = run[2 * N + i];
  if (count_col >= 0) cnt += (double)row[count_col] >= thresh ? 1.0 : 0.0;   // NaN >= thresh is false
  bool ok = isfinite(ret);
  double term[B2Q_ES_MAX_TERMS];
#pragma unroll
  for (int j = 0; j < B2Q_ES_MAX_TERMS; j++)
    if (j < ncols) { term[j] = run[(3 + j) * N + i] + (double)row[cols.c[j]]; ok = ok && isfinite(term[j]); }
  if (!done[i]) {
    run[i] = ret; run[N + i] = len; run[2 * N + i] = cnt;
#pragma unroll
    for (int j = 0; j < B2Q_ES_MAX_TERMS; j++)
      if (j < ncols) run[(3 + j) * N + i] = term[j];
    return;
  }
  // the episode ends: fold it into the window (or only count it, when a sum is not finite) and start the next one from zero
  if (ok) {
    win[i] += 1.0;
    win[2 * N + i] += ret;
    win[3 * N + i] += len;
    if (count_col >= 0) win[4 * N + i] += cnt / len;
#pragma unroll
    for (int j = 0; j < B2Q_ES_MAX_TERMS; j++)
      if (j < ncols) { win[(5 + j) * N + i] += term[j]; win[(5 + ncols + j) * N + i] += term[j] / len; }
  } else {
    win[N + i] += 1.0;
  }
  run[i] = 0.0; run[N + i] = 0.0; run[2 * N + i] = 0.0;
#pragma unroll
  for (int j = 0; j < B2Q_ES_MAX_TERMS; j++)
    if (j < ncols) run[(3 + j) * N + i] = 0.0;
}

// one warp per individual: deterministic shuffle-tree sum over its `rollouts` consecutive envs
template <typename T>
__global__ void es_fitness_kernel(const T* __restrict__ ret, const int32_t* __restrict__ len, T* __restrict__ fitness, T* __restrict__ mean_len,
                                  int pop, int rollouts) {
  int ind = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (ind >= pop) return;
  T s = 0, l = 0;
  for (int r = lane; r < rollouts; r += 32) { s += ret[(size_t)ind * rollouts + r]; l += (T)len[(size_t)ind * rollouts + r]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); l += __shfl_xor_sync(0xffffffffu, l, o); }
  if (lane == 0) { fitness[ind] = s / (T)rollouts; if (mean_len) mean_len[ind] = l / (T)rollouts; }
}

}  // namespace

extern "C" {

int b2q_es_accumulate(const void* reward, const uint8_t* done, uint8_t* alive, void* ret, int32_t* len, int n, int elem_size, void* stream) {
  if (!reward || !done || !alive || !ret || !len || n < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  if (elem_size == 4) es_accumulate_kernel<float><<<(n + 255) / 256, 256, 0, s>>>((const float*)reward, done, alive, (float*)ret, len, n);
  else es_accumulate_kernel<double><<<(n + 255) / 256, 256, 0, s>>>((const double*)reward, done, alive, (double*)ret, len, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int b2q_es_accumulate_terms(const void* reward, const uint8_t* done, uint8_t* alive, void* ret, int32_t* len, const void* info, int info_dim,
                            const int32_t* cols, int ncols, void* term_sum, int count_col, double thresh, int32_t* count, int n, int elem_size,
                            void* stream) {
  if (!reward || !done || !alive || !ret || !len || n < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  if (ncols < 0 || ncols > B2Q_ES_MAX_TERMS || count_col < -1) return -1;
  if ((ncols > 0 || count_col >= 0) && (!info || info_dim < 1)) return -1;
  if ((ncols > 0 && (!cols || !term_sum)) || (count_col >= 0 && (!count || count_col >= info_dim))) return -1;
  TermCols tc = {};
  for (int j = 0; j < ncols; j++) {
    if (cols[j] < 0 || cols[j] >= info_dim) return -1;
    tc.c[j] = cols[j];
  }
  cudaStream_t s = (cudaStream_t)stream;
  int blocks = (n + 255) / 256;
  if (elem_size == 4)
    es_accumulate_terms_kernel<float><<<blocks, 256, 0, s>>>((const float*)reward, done, alive, (float*)ret, len, (const float*)info, info_dim, tc, ncols,
                                                             (float*)term_sum, count_col, (float)thresh, count, n);
  else
    es_accumulate_terms_kernel<double><<<blocks, 256, 0, s>>>((const double*)reward, done, alive, (double*)ret, len, (const double*)info, info_dim, tc,
                                                              ncols, (double*)term_sum, count_col, thresh, count, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int b2q_train_episode_stats(const void* reward, const uint8_t* done, const void* info, int info_dim, const int32_t* cols, int ncols, int count_col,
                            double thresh, double* run, double* win, int n, int elem_size, void* stream) {
  if (!reward || !done || !run || !win || n < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  if (ncols < 0 || ncols > B2Q_ES_MAX_TERMS || count_col < -1) return -1;
  if ((ncols > 0 || count_col >= 0) && (!info || info_dim < 1)) return -1;
  if ((ncols > 0 && !cols) || count_col >= info_dim) return -1;
  TermCols tc = {};
  for (int j = 0; j < ncols; j++) {
    if (cols[j] < 0 || cols[j] >= info_dim) return -1;
    tc.c[j] = cols[j];
  }
  cudaStream_t s = (cudaStream_t)stream;
  int blocks = (n + 255) / 256;
  if (elem_size == 4)
    train_episode_stats_kernel<float><<<blocks, 256, 0, s>>>((const float*)reward, done, (const float*)info, info_dim, tc, ncols, count_col, thresh,
                                                             run, win, n);
  else
    train_episode_stats_kernel<double><<<blocks, 256, 0, s>>>((const double*)reward, done, (const double*)info, info_dim, tc, ncols, count_col, thresh,
                                                              run, win, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int b2q_es_fitness(const void* ret, const int32_t* len, void* fitness, void* mean_len, int pop, int rollouts, int elem_size, void* stream) {
  if (!ret || !len || !fitness || pop < 1 || rollouts < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  int threads = 128, blocks = (pop * 32 + threads - 1) / threads;
  if (elem_size == 4) es_fitness_kernel<float><<<blocks, threads, 0, s>>>((const float*)ret, len, (float*)fitness, (float*)mean_len, pop, rollouts);
  else es_fitness_kernel<double><<<blocks, threads, 0, s>>>((const double*)ret, len, (double*)fitness, (double*)mean_len, pop, rollouts);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// §8f-1: batched ETG weight fit on the device.  One thread per ES individual restates Opt_with_points + LS_sol
// (train.py:59-110): two gradient-descent least-squares solves (<= 1000 iterations, step 0.05, Tikhonov pull towards w0)
// of a 6x20 system, in float64 like the NumPy reference.  obs6x20 = ETG features at the six control-point times.
namespace {
__device__ void ls_sol_dev(const double* A /*6x20*/, const double* bvec /*6*/, const double* w0 /*20*/, double lamb, double precision, double alpha, double* x /*20 out*/) {
  double AtA[20][20], Atb[20];
  for (int i = 0; i < 20; i++) {
    double s = 0; for (int r = 0; r < 6; r++) s += A[r * 20 + i] * bvec[r];
    Atb[i] = s;
    for (int j = 0; j < 20; j++) { double t = 0; for (int r = 0; r < 6; r++) t += A[r * 20 + i] * A[r * 20 + j]; AtA[i][j] = t; }
  }
  for (int i = 0; i < 20; i++) x[i] = w0[i];
  auto sqerr = [&]() { double e = 0; for (int r = 0; r < 6; r++) { double s = -bvec[r]; for (int i = 0; i < 20; i++) s += A[r * 20 + i] * x[i]; e += s * s; } return e; };
  double err = sqerr();
  int it = 0;
  while (err > precision && it < 1000) {
    double dx[20];
    for (int i = 0; i < 20; i++) { double s = -Atb[i]; for (int j = 0; j < 20; j++) s += AtA[i][j] * x[j]; dx[i] = s + lamb * (x[i] - w0[i]); }
    for (int i = 0; i < 20; i++) x[i] -= alpha * dx[i];
    err = sqerr();
    it++;
  }
}
__global__ void etg_fit_kernel(const double* __restrict__ obs6x20, const double* __restrict__ prior_points /*6x2*/, const double* __restrict__ solutions /*[pop][12]*/,
                               const double* __restrict__ w0 /*3x20*/, const double* __restrict__ b0 /*3*/, double lamb, double precision,
                               double* __restrict__ w_out /*[pop][3][20]*/, double* __restrict__ b_out /*[pop][3]*/, int pop) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pop) return;
  double A[120];
  for (int k = 0; k < 120; k++) A[k] = obs6x20[k];
  double bx = b0[0], bz = b0[2], px[6], pz[6];
  for (int r = 0; r < 6; r++) {   // points = prior_points + solution.reshape(-1,2); points_t = points - b   (train.py:405-406,97)
    px[r] = prior_points[2 * r] + solutions[(size_t)i * 12 + 2 * r] - bx;
    pz[r] = prior_points[2 * r + 1] + solutions[(size_t)i * 12 + 2 * r + 1] - bz;
  }
  double x1[20], x2[20];
  ls_sol_dev(A, px, w0, lamb, precision, 0.05, x1);
  ls_sol_dev(A, pz, w0 + 40, lamb, precision, 0.05, x2);
  for (int h = 0; h < 20; h++) { w_out[(size_t)i * 60 + h] = x1[h]; w_out[(size_t)i * 60 + 20 + h] = 0.0; w_out[(size_t)i * 60 + 40 + h] = x2[h]; }
  b_out[(size_t)i * 3] = bx; b_out[(size_t)i * 3 + 1] = 0.0; b_out[(size_t)i * 3 + 2] = bz;
}
}  // namespace

extern "C" int b2q_etg_fit(const double* obs6x20, const double* prior_points, const double* solutions, const double* w0, const double* b0, double lamb,
                           double precision, double* w_out, double* b_out, int pop, void* stream) {
  if (!obs6x20 || !prior_points || !solutions || !w0 || !b0 || !w_out || !b_out || pop < 1) return -1;
  etg_fit_kernel<<<(pop + 31) / 32, 32, 0, (cudaStream_t)stream>>>(obs6x20, prior_points, solutions, w0, b0, lamb, precision, w_out, b_out, pop);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// ---------------------------------------------------------------------------------------------------------------------
// §8f-4: dynamics-identification fitness (model/Dynamic_parallel_model.py:29-41,53-68).  Per env and control step the
// squared, std-normalised deviation of the 12 joint angles and 3 body rates from the recorded real-robot statistics is
// accumulated; the episode reward is 30 - (max_j mean_t motor + max_k mean_t drpy) / 2.
namespace {
template <typename T>
__global__ void dyn_accum_kernel(const T* __restrict__ info /*[N][56]*/, const T* __restrict__ mean15 /*motor12|drpy3 at this step*/, const T* __restrict__ std15,
                                 T* __restrict__ acc /*[N][15]*/, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 15) return;
  int e = i / 15, c = i % 15;
  T x = c < 12 ? info[(size_t)e * 56 + 42 + c] : info[(size_t)e * 56 + 39 + (c - 12)];   // joint_angle | obs-IMU[3:] (info columns, include/b2q.h)
  T d = x - mean15[c], s = std15[c];
  acc[i] += d * d / (s * s);
}
// max that propagates NaN like the reference's np.max (fmax drops it: a NaN column would leave a finite reward from the other 14)
template <typename T>
__device__ __forceinline__ T max_nan(T a, T b) { return (a != a || a > b) ? a : b; }
template <typename T>
__global__ void dyn_finish_kernel(const T* __restrict__ acc, int steps, T* __restrict__ reward, int n) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  T lm = acc[(size_t)e * 15], ld = acc[(size_t)e * 15 + 12];
  for (int c = 1; c < 12; c++) lm = max_nan(lm, acc[(size_t)e * 15 + c]);
  for (int c = 13; c < 15; c++) ld = max_nan(ld, acc[(size_t)e * 15 + c]);
  reward[e] = T(30) - (lm / T(steps) + ld / T(steps)) / T(2);
}
}  // namespace

extern "C" {
int b2q_dyn_accumulate(const void* info, const void* mean15, const void* std15, void* acc, int n, int elem_size, void* stream) {
  if (!info || !mean15 || !std15 || !acc || n < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  int blocks = (n * 15 + 255) / 256;
  if (elem_size == 4) dyn_accum_kernel<float><<<blocks, 256, 0, s>>>((const float*)info, (const float*)mean15, (const float*)std15, (float*)acc, n);
  else dyn_accum_kernel<double><<<blocks, 256, 0, s>>>((const double*)info, (const double*)mean15, (const double*)std15, (double*)acc, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_dyn_finish(const void* acc, int steps, void* reward, int n, int elem_size, void* stream) {
  if (!acc || !reward || n < 1 || steps < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  if (elem_size == 4) dyn_finish_kernel<float><<<(n + 255) / 256, 256, 0, s>>>((const float*)acc, steps, (float*)reward, n);
  else dyn_finish_kernel<double><<<(n + 255) / 256, 256, 0, s>>>((const double*)acc, steps, (double*)reward, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
}
