// b2q_deploy.cu — the deployment-rehearsal kernels (include/b2q_deploy.h): the table-driven observation ETG block and action of the
// reference's deployment/test.py:93-99, one thread per (env, joint column), the table row taken from the handle's per-env step counter.
#include <cuda_runtime.h>
#include <string>
#include "b2q_sim.cuh"
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

}  // extern "C"
