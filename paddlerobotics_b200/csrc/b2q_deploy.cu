// b2q_deploy.cu — the deployment-rehearsal kernels (include/b2q_deploy.h): the table-driven observation ETG block and action of the
// reference's deployment/test.py:93-99, one thread per (env, joint column), the table row taken from the handle's per-env step counter;
// and the open-loop Bezier gait of --gait 1 (b2q_bezier.h), one thread per env.
#include <cuda_runtime.h>
#include <string>
#include "b2q_sim.cuh"
#include "b2q_bezier.h"
#include "b2q_env_view.h"
#include "../../include/b2q_deploy.h"

namespace b2q {
namespace {

template <typename T> __device__ __forceinline__ T quiet_nan();
template <> __device__ __forceinline__ float quiet_nan<float>() { return __int_as_float(0x7fc00000); }
template <> __device__ __forceinline__ double quiet_nan<double>() { return __longlong_as_double(0x7ff8000000000000LL); }
// one rounding per operation, as NumPy's a * b + c: the compiler would otherwise contract the pair into a fused multiply-add
__device__ __forceinline__ float mul_add_rn(float a, float b, float c) { return __fadd_rn(__fmul_rn(a, b), c); }
__device__ __forceinline__ double mul_add_rn(double a, double b, double c) { return __dadd_rn(__dmul_rn(a, b), c); }

template <typename T>
__global__ void deploy_obs_kernel(const Model<T>* __restrict__ md, const int32_t* __restrict__ step_count, const T* __restrict__ table, int rows,
                                  int etg_col, int normal, T* __restrict__ obs, int obs_dim, T* __restrict__ rec, int rec_rows, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 12) return;
  const int e = i / 12, c = i - e * 12;
  const int r = step_count[e];
  T v = (r >= 0 && r < rows) ? table[(size_t)r * 12 + c] : quiet_nan<T>();   // past the table: NaN, never a read outside it
  if (normal) v = (v - md->etg_mean[c]) * md->etg_istd[c];                    // write_obs's expression (b2q_sim.cuh)
  T* row = obs + (size_t)e * obs_dim;
  if (etg_col >= 0) row[etg_col + c] = v;
  if (rec && e == 0 && r >= 0 && r < rec_rows) {   // env 0's 12 threads copy its row: thread c the columns c, c + 12, ...
    T* dst = rec + (size_t)r * obs_dim;
    for (int j = c; j < obs_dim; j += 12)
      if (etg_col < 0 || j < etg_col || j >= etg_col + 12) dst[j] = row[j];   // the ETG columns are this launch's own values
    if (etg_col >= 0) dst[etg_col + c] = v;
  }
}

template <typename T>
__global__ void deploy_act_kernel(const int32_t* __restrict__ step_count, const float* __restrict__ pol, T bound, const T* __restrict__ table, int rows,
                                  T* __restrict__ action, T* __restrict__ rec, int rec_rows, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 12) return;
  const int e = i / 12, c = i - e * 12;
  const int r = step_count[e];
  const T a = (r >= 0 && r < rows) ? mul_add_rn(bound, (T)pol[i], table[(size_t)r * 12 + c]) : quiet_nan<T>();
  action[i] = a;
  if (rec && e == 0 && r >= 0 && r < rec_rows) rec[(size_t)r * 12 + c] = a;
}

// GaitWrapper.reset (EnvWrapper.py:140-153): the feet of each env's current joint angles and a fresh gait clock
template <typename T>
__global__ void bezier_reset_kernel(const P4<T>* __restrict__ st, double* __restrict__ gait, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  double q[12];
  for (int k = 0; k < 4; k++) {
    const P4<T> p = ldp(st, 4 + k, n, e);
    q[3 * k] = (double)p.x; q[3 * k + 1] = (double)p.y; q[3 * k + 2] = (double)p.z;
  }
  double s[bezier::BEZ_K];
  bezier::reset_env(q, s);
  for (int j = 0; j < bezier::BEZ_K; j++) gait[(size_t)e * bezier::BEZ_K + j] = s[j];
}

// GaitWrapper.step (EnvWrapper.py:155-191) at each env's step counter r: timesteps = r + 1, the reference foot's contact bit from the
// observation the student saw, and action += IK(feet) - POSE_ORI with the increment rounded once to T
template <typename T>
__global__ void bezier_act_kernel(const int32_t* __restrict__ step_count, double* __restrict__ gait, const T* __restrict__ obs, int obs_dim,
                                  int contact_col, T* __restrict__ action, double* __restrict__ rec_feet, int rec_rows, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int r = step_count[e];
  double s[bezier::BEZ_K], feet[12], ang[12];
  for (int j = 0; j < bezier::BEZ_K; j++) s[j] = gait[(size_t)e * bezier::BEZ_K + j];
  bezier::act_env(s, r + 1, obs[(size_t)e * obs_dim + contact_col] == T(1), feet, ang);
  for (int j = 0; j < bezier::BEZ_K; j++) gait[(size_t)e * bezier::BEZ_K + j] = s[j];
  T* a = action + (size_t)e * 12;
  for (int j = 0; j < 12; j++) a[j] = a[j] + (T)(ang[j] - bezier::pose_ori(j % 3));
  if (rec_feet && e == 0 && r >= 0 && r < rec_rows)
    for (int j = 0; j < 12; j++) rec_feet[(size_t)r * 12 + j] = feet[j];
}

int fail(B2QHandle h, const char* msg) { env_set_error(h, msg); return B2Q_EINVAL; }

int on_device(B2QHandle h, int device) {
  int cur = -1;
  if (cudaGetDevice(&cur) == cudaSuccess && cur == device) return B2Q_OK;
  if (cudaSetDevice(device) != cudaSuccess) { env_set_error(h, "cudaSetDevice failed"); return B2Q_ECUDA; }
  return B2Q_OK;
}

int launched(B2QHandle h, const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return B2Q_OK;
  env_set_error(h, (std::string(what) + ": " + cudaGetErrorString(e)).c_str());
  return B2Q_ECUDA;
}

}  // namespace
}  // namespace b2q

using namespace b2q;

extern "C" {

int b2q_deploy_obs(B2QHandle h, const void* table, int rows, int etg_col, int normal, void* obs, void* rec_obs, int rec_rows, void* stream) {
  EnvView v;
  if (env_view(h, &v) != B2Q_OK) return B2Q_EINVAL;
  if (!table || !obs) return fail(h, "b2q_deploy_obs: null table or obs");
  if (rows < 1) return fail(h, "b2q_deploy_obs: rows must be >= 1");
  if (etg_col < -1 || etg_col > v.obs_dim - 12) return fail(h, "b2q_deploy_obs: etg_col must be -1 or in [0, obs_dim - 12]");
  if (rec_obs && rec_rows < 1) return fail(h, "b2q_deploy_obs: rec_rows must be >= 1 when rec_obs is given");
  if (int rc = on_device(h, v.device)) return rc;
  const int blocks = (v.N * 12 + 255) / 256;
  cudaStream_t s = (cudaStream_t)stream;
  if (v.elem_size == 4)
    deploy_obs_kernel<float><<<blocks, 256, 0, s>>>((const Model<float>*)v.model, v.step_count, (const float*)table, rows, etg_col, normal, (float*)obs,
                                                    v.obs_dim, (float*)rec_obs, rec_rows, v.N);
  else
    deploy_obs_kernel<double><<<blocks, 256, 0, s>>>((const Model<double>*)v.model, v.step_count, (const double*)table, rows, etg_col, normal, (double*)obs,
                                                     v.obs_dim, (double*)rec_obs, rec_rows, v.N);
  return launched(h, "b2q_deploy_obs");
}

int b2q_deploy_act(B2QHandle h, const float* policy_out, double act_bound, const void* table, int rows, void* action, void* rec_act, int rec_rows,
                   void* stream) {
  EnvView v;
  if (env_view(h, &v) != B2Q_OK) return B2Q_EINVAL;
  if (!policy_out || !table || !action) return fail(h, "b2q_deploy_act: null policy_out, table or action");
  if (rows < 1) return fail(h, "b2q_deploy_act: rows must be >= 1");
  if (rec_act && rec_rows < 1) return fail(h, "b2q_deploy_act: rec_rows must be >= 1 when rec_act is given");
  if (int rc = on_device(h, v.device)) return rc;
  const int blocks = (v.N * 12 + 255) / 256;
  cudaStream_t s = (cudaStream_t)stream;
  if (v.elem_size == 4)
    deploy_act_kernel<float><<<blocks, 256, 0, s>>>(v.step_count, policy_out, (float)act_bound, (const float*)table, rows, (float*)action, (float*)rec_act,
                                                    rec_rows, v.N);
  else
    deploy_act_kernel<double><<<blocks, 256, 0, s>>>(v.step_count, policy_out, act_bound, (const double*)table, rows, (double*)action, (double*)rec_act,
                                                     rec_rows, v.N);
  return launched(h, "b2q_deploy_act");
}

int b2q_bezier_reset(B2QHandle h, void* state, void* stream) {
  EnvView v;
  if (env_view(h, &v) != B2Q_OK) return B2Q_EINVAL;
  if (v.etg_enabled) return fail(h, "b2q_bezier_reset: the handle must be created with etg_enabled = 0");
  if (!state) return fail(h, "b2q_bezier_reset: null state");
  if (int rc = on_device(h, v.device)) return rc;
  const int blocks = (v.N + 127) / 128;
  cudaStream_t s = (cudaStream_t)stream;
  if (v.elem_size == 4)
    bezier_reset_kernel<float><<<blocks, 128, 0, s>>>((const P4<float>*)v.state, (double*)state, v.N);
  else
    bezier_reset_kernel<double><<<blocks, 128, 0, s>>>((const P4<double>*)v.state, (double*)state, v.N);
  return launched(h, "b2q_bezier_reset");
}

int b2q_bezier_act(B2QHandle h, void* state, int contact_col, const void* obs, void* action, double* rec_feet, int rec_rows, void* stream) {
  EnvView v;
  if (env_view(h, &v) != B2Q_OK) return B2Q_EINVAL;
  if (v.etg_enabled) return fail(h, "b2q_bezier_act: the handle must be created with etg_enabled = 0");
  if (!state || !obs || !action) return fail(h, "b2q_bezier_act: null state, obs or action");
  if (contact_col < 0 || contact_col >= v.obs_dim) return fail(h, "b2q_bezier_act: contact_col must be in [0, obs_dim)");
  if (rec_feet && rec_rows < 1) return fail(h, "b2q_bezier_act: rec_rows must be >= 1 when rec_feet is given");
  if (int rc = on_device(h, v.device)) return rc;
  // one warp per block: 4096 envs are only 128 warps, spread over the SMs rather than packed four to an SM
  const int blocks = (v.N + 31) / 32;
  cudaStream_t s = (cudaStream_t)stream;
  if (v.elem_size == 4)
    bezier_act_kernel<float><<<blocks, 32, 0, s>>>(v.step_count, (double*)state, (const float*)obs, v.obs_dim, contact_col, (float*)action,
                                                    rec_feet, rec_rows, v.N);
  else
    bezier_act_kernel<double><<<blocks, 32, 0, s>>>(v.step_count, (double*)state, (const double*)obs, v.obs_dim, contact_col, (double*)action,
                                                     rec_feet, rec_rows, v.N);
  return launched(h, "b2q_bezier_act");
}

}  // extern "C"
