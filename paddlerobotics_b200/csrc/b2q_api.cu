// b2q_api.cu — sm_90a kernels and the C ABI (include/b2q.h) of the batched A1 simulator.
//
// Kernel map (SURVEY.md §7): K1 b2q_step_kernel (hot: R fused physics substeps + ETG + obs/reward pack, optional
// in-kernel auto-reset), K2 b2q_reset_kernel (masked snapshot copy), b2q_settle_kernel (builds the snapshot), and
// small repack kernels.  Mapping: one lane per leg, 4 lanes per robot, 8 robots per warp; SoA float4 packs in HBM
// ([pack][env]) so that every lane's 16-byte load is part of a fully coalesced 128-byte warp transaction.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <new>
#include <string>
#include "b2q_host_common.h"
#include "b2q_env_view.h"
#include "b2q_render_internal.h"
#include "b2q_snapshot.h"
#include "../../include/b2q_render.h"

using namespace b2q;

namespace {

struct WarpComm {
  int k;
  unsigned char* scr;   // this robot's shared-memory scratch, scratch_floats(FEAT) elements (null in the reset kernel)
  __device__ __forceinline__ int leg() const { return k; }
  template <typename T> __device__ __forceinline__ T* scratch() const { return reinterpret_cast<T*>(scr); }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ bool any(bool f) const { return __any_sync(0xffffffffu, f) != 0; }   // over the whole warp (8 robots)
  template <typename T>
  __device__ __forceinline__ T sum4(T v) const {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    return v;
  }
  template <typename T>
  __device__ __forceinline__ T bcast(T v, int f) const { return __shfl_sync(0xffffffffu, v, f, 4); }
#ifdef B2Q_REGION_CLOCKS
  mutable long long t_mark = 0, cyc[RC_N] = {};   // cycles per region of this launch, in registers (every index is a constant)
  __device__ __forceinline__ void mark(int region) const { const long long t = clock64(); cyc[region] += t - t_mark; t_mark = t; }
#endif
};

#ifdef B2Q_REGION_CLOCKS
// one row per warp of the step kernel, summed over launches: the RC_N region cycles, the entry-to-exit cycles and the launch count
constexpr int RC_MAX_WARPS = 8192, RC_COLS = RC_N + 2;
__device__ unsigned long long g_region_clocks[RC_MAX_WARPS][RC_COLS];
#endif

template <typename T>
__device__ __forceinline__ const Model<T>& stage_model(const Model<T>* g, unsigned char* smem) {
  // model constants (~1 KB) staged once per CTA in shared memory: lanes of different legs read different
  // LegModel rows, which a __constant__ bank would serialise
  // 128-bit loads, four per thread in flight before the first store: one memory latency instead of a 13-deep chain of dependent 4-byte
  // load -> store pairs per 32-thread CTA (2 us of the 115 us step in the round-2 profile).  The device copy is padded to a multiple of 16 bytes.
  Model<T>* s = reinterpret_cast<Model<T>*>(smem);
  const uint4* src = reinterpret_cast<const uint4*>(g);
  uint4* dst = reinterpret_cast<uint4*>(s);
  constexpr int NV = (int)((sizeof(Model<T>) + 15) / 16);
  for (int i0 = threadIdx.x; i0 < NV; i0 += 4 * blockDim.x) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { const int i = i0 + k * (int)blockDim.x; if (i < NV) v[k] = __ldg(src + i); }
#pragma unroll
    for (int k = 0; k < 4; k++) { const int i = i0 + k * (int)blockDim.x; if (i < NV) dst[i] = v[k]; }
  }
  __syncthreads();
  return *s;
}

// staged block (shared memory) -> global / pinned host memory: 128-bit stores when both ends are 16-byte aligned (full CTAs always are:
// 8 rows x 49 or 56 floats), scalar otherwise
template <typename T>
__device__ __forceinline__ void copy_block(T* __restrict__ dst, const T* stage, int n) {
  constexpr int PER = 16 / (int)sizeof(T);
  if ((((size_t)dst | (size_t)stage) & 15) == 0 && n % PER == 0) {
    uint4* d4 = reinterpret_cast<uint4*>(dst); const uint4* s4 = reinterpret_cast<const uint4*>(stage);
    for (int i = threadIdx.x; i < n / PER; i += blockDim.x) d4[i] = s4[i];
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = stage[i];
  }
}

// the CTA's staged 49-wide rows -> the caller's [N][obs_dim] array (sensor_mode selection applied), coalesced
template <typename T>
__device__ __forceinline__ void emit_obs_block(const Model<T>& md, const T* stage, T* __restrict__ obs, int env0, int rows) {
  const int od = md.obs_dim;
  T* dst = obs + (size_t)env0 * od;
  if (md.obs_identity) { copy_block(dst, stage, rows * OBS_DIM); return; }
  for (int i = threadIdx.x; i < rows * od; i += blockDim.x) { int r = i / od, j = i - r * od; dst[i] = obs_out_elem(md, stage + r * OBS_DIM, j); }
}

// Terrain atlas (b2q_set_terrain_tiles): T height-field tiles on the handle's one hf_* grid, and the tile each env reads.  The TILES = 1
// bodies below load env i's tile once per launch and step or settle it on a Cfg whose `hf` is that tile's base pointer (a 64-bit offset),
// so terrain_height runs unchanged and env i computes what a plain height-field handle built on tile tile_of_env[i] computes.  They are
// kernels of their own (b2q_step_tiles_kernel, b2q_settle_tiles_kernel): the default kernels' code does not change.
struct Tiles {
  const int32_t* tile_of_env;   // [N]
  long long tile_elems;         // hf_nx * hf_ny
};
template <typename T, int TILES>
__device__ __forceinline__ Cfg<T> env_cfg(const Cfg<T>& cf, const Tiles& tl, int env) {
  Cfg<T> c = cf;
  if constexpr (TILES != 0) c.hf = cf.hf + (size_t)tl.tile_of_env[env] * (size_t)tl.tile_elems;
  return c;
}

template <typename T, int FEAT, int TILES>
__device__ __forceinline__ void step_cta(const Cfg<T>& cf, const Tiles& tl, const Model<T>* __restrict__ gm, const Buffers<T>& B, const T* __restrict__ action,
                                         int donef, int auto_reset, T* __restrict__ obs, T* __restrict__ reward, uint8_t* __restrict__ done, T* __restrict__ info) {
#ifdef B2Q_REGION_CLOCKS
  const long long t_entry = clock64();
#endif
  extern __shared__ __align__(32) unsigned char smem[];
  const Model<T>& md = stage_model(gm, smem);
  // the CTA's observation rows are contiguous in [N][OBS_DIM]: stage them in shared memory and store the block with
  // full-width coalesced stores (the lanes produce the row in 3-element pieces; `obs` may be pinned HOST memory, where
  // piecewise stores would each become a small PCIe write)
  T* stage = reinterpret_cast<T*>(smem + ((sizeof(Model<T>) + 31) & ~size_t(31)));
  int gid = blockIdx.x * blockDim.x + threadIdx.x;
  int env = gid >> 2;
  const int env0 = (blockIdx.x * blockDim.x) >> 2, per_cta = blockDim.x >> 2;
  bool valid = env < B.N;
  // whole warps stay convergent for the shuffles; invalid lanes (ragged last CTA) redo the CTA's first robot in their own staging
  // row and never store to global memory
  const int srow = env0 + (int)(threadIdx.x >> 2);
  if (!valid) env = B.N - 1;
  T* istage0 = stage + (size_t)per_cta * OBS_DIM;
  WarpComm cm{(int)(threadIdx.x & 3), reinterpret_cast<unsigned char*>(istage0 + (size_t)per_cta * INFO_DIM + (size_t)(threadIdx.x >> 2) * scratch_floats(FEAT))};
  // the info rows (56 floats per env, produced in 3-float pieces) are staged the same way: one coalesced block per CTA, so that `info`
  // too may be pinned HOST memory (train.py:150-157 reads info every step)
  T* istage = istage0;
#ifdef B2Q_REGION_CLOCKS
  cm.t_mark = t_entry;
#endif
  if constexpr (TILES != 0) {
    step_lane<T, FEAT>(cm, env_cfg<T, TILES>(cf, tl, env), md, B, env, valid, action, donef, auto_reset, stage + (ptrdiff_t)(srow - env) * OBS_DIM, reward, done, istage,
                       env0, env0);
  } else {
    step_lane<T, FEAT>(cm, cf, md, B, env, valid, action, donef, auto_reset, stage + (ptrdiff_t)(srow - env) * OBS_DIM, reward, done, istage, env0, env0);
  }
  __syncthreads();
  const int rows = min(per_cta, B.N - env0);
  emit_obs_block(md, stage, obs, env0, rows);
  copy_block(info + (size_t)env0 * INFO_DIM, istage, rows * INFO_DIM);
#ifdef B2Q_REGION_CLOCKS
  B2Q_MARK(cm, RC_EPILOGUE);
  const int warp = (int)(gid >> 5);
  if ((threadIdx.x & 31) == 0 && warp < RC_MAX_WARPS) {   // launches on one stream run one after another: plain read-modify-write
#pragma unroll
    for (int r = 0; r < RC_N; r++) g_region_clocks[warp][r] += (unsigned long long)cm.cyc[r];
    g_region_clocks[warp][RC_N] += (unsigned long long)(cm.t_mark - t_entry);
    g_region_clocks[warp][RC_N + 1] += 1;
  }
#endif
}

template <typename T, int FEAT>
__global__ void __launch_bounds__(128) b2q_step_kernel(Cfg<T> cf, const Model<T>* __restrict__ gm, Buffers<T> B, const T* __restrict__ action, int donef,
                                                       int auto_reset, T* __restrict__ obs, T* __restrict__ reward, uint8_t* __restrict__ done, T* __restrict__ info) {
  step_cta<T, FEAT, 0>(cf, Tiles{nullptr, 0}, gm, B, action, donef, auto_reset, obs, reward, done, info);
}
template <typename T, int FEAT>
__global__ void __launch_bounds__(128) b2q_step_tiles_kernel(Cfg<T> cf, Tiles tl, const Model<T>* __restrict__ gm, Buffers<T> B, const T* __restrict__ action,
                                                             int donef, int auto_reset, T* __restrict__ obs, T* __restrict__ reward, uint8_t* __restrict__ done,
                                                             T* __restrict__ info) {
  step_cta<T, FEAT, 1>(cf, tl, gm, B, action, donef, auto_reset, obs, reward, done, info);
}

template <typename T, int FEAT, int TILES>
__device__ __forceinline__ void settle_cta(const Cfg<T>& cf, const Tiles& tl, const Model<T>* __restrict__ gm, const Buffers<T>& B, const uint8_t* __restrict__ mask) {
  extern __shared__ __align__(32) unsigned char smem[];
  const Model<T>& md = stage_model(gm, smem);
  int gid = blockIdx.x * blockDim.x + threadIdx.x;
  int env = gid >> 2;
  bool valid = env < B.N;
  if (!valid) env = B.N - 1;
  if (mask && !mask[env]) valid = false;
  T* scr0 = reinterpret_cast<T*>(smem + ((sizeof(Model<T>) + 31) & ~size_t(31))) + (size_t)(blockDim.x >> 2) * (OBS_DIM + INFO_DIM);
  WarpComm cm{(int)(threadIdx.x & 3), reinterpret_cast<unsigned char*>(scr0 + (size_t)(threadIdx.x >> 2) * scratch_floats(FEAT))};
  if constexpr (TILES != 0) settle_lane<T, FEAT>(cm, env_cfg<T, TILES>(cf, tl, env), md, B, env, valid);
  else settle_lane<T, FEAT>(cm, cf, md, B, env, valid);
}

template <typename T, int FEAT>
__global__ void __launch_bounds__(128) b2q_settle_kernel(Cfg<T> cf, const Model<T>* __restrict__ gm, Buffers<T> B, const uint8_t* __restrict__ mask) {
  settle_cta<T, FEAT, 0>(cf, Tiles{nullptr, 0}, gm, B, mask);
}
template <typename T, int FEAT>
__global__ void __launch_bounds__(128) b2q_settle_tiles_kernel(Cfg<T> cf, Tiles tl, const Model<T>* __restrict__ gm, Buffers<T> B, const uint8_t* __restrict__ mask) {
  settle_cta<T, FEAT, 1>(cf, tl, gm, B, mask);
}

template <typename T>
__global__ void __launch_bounds__(128) b2q_reset_kernel(Cfg<T> cf, const Model<T>* __restrict__ gm, Buffers<T> B, const uint8_t* __restrict__ mask, const T* __restrict__ xoff,
                                                        T* __restrict__ obs) {
  extern __shared__ __align__(32) unsigned char smem[];
  const Model<T>& md = stage_model(gm, smem);
  T* stage = reinterpret_cast<T*>(smem + ((sizeof(Model<T>) + 31) & ~size_t(31)));
  int gid = blockIdx.x * blockDim.x + threadIdx.x;
  int env = gid >> 2;
  const int env0 = (blockIdx.x * blockDim.x) >> 2;
  bool valid = env < B.N;
  if (!valid) env = B.N - 1;
  if (mask && !mask[env]) valid = false;
  WarpComm cm{(int)(threadIdx.x & 3), nullptr};
  T* srow = stage + (size_t)(threadIdx.x >> 2) * OBS_DIM;
  reset_lane<T>(cm, cf, md, B, env, valid, obs ? srow : (T*)nullptr, xoff);
  if (obs) {   // masked-out envs keep their previous observation row
    __syncwarp();
    if (valid) { const int od = md.obs_dim; for (int j = threadIdx.x & 3; j < od; j += 4) obs[(size_t)env * od + j] = obs_out_elem(md, srow, j); }
  }
  (void)env0;
}

template <typename T>
__global__ void b2q_pack_param_kernel(const T* __restrict__ dyn, const T* __restrict__ def48, P4<T>* param, const uint8_t* __restrict__ mask, int N, T max_latency,
                                      int* __restrict__ overflow) {
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= N || (mask && !mask[env])) return;
  pack_param_env<T>(dyn, def48, param, N, env);
  const T lat = dyn ? dyn[(size_t)env * 48 + 25] : def48[25];
  if (!(lat <= max_latency)) atomicMax(overflow, 1);   // control latency beyond the observation ring: refuse instead of clamping silently
}
template <typename T>
__global__ void b2q_pack_force_kernel(const T* __restrict__ f, P4<T>* extf, int N) {
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= N) return;
  P4<T> p; p.x = f ? f[(size_t)env * 3] : T(0); p.y = f ? f[(size_t)env * 3 + 1] : T(0); p.z = f ? f[(size_t)env * 3 + 2] : T(0); p.w = T(0);
  extf[env] = p;
}
template <typename T>
__global__ void b2q_pack_etg_kernel(const T* __restrict__ w, const T* __restrict__ b, P4<T>* etg, const uint8_t* __restrict__ mask, int N) {
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= N || (mask && !mask[env])) return;
  pack_etg_env<T>(w, b, etg, N, env);
}
template <typename T>
__global__ void b2q_get_state_kernel(const P4<T>* st, T* out, int N) {
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env < N) get_state_env<T>(st, out, N, env);
}
template <typename T>
__global__ void b2q_set_state_kernel(P4<T>* st, const T* in, int N) {
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env < N) set_state_env<T>(st, in, N, env);
}

thread_local std::string g_create_err;

// ---- env snapshot (b2q_snapshot_*): header + the whole SoA pool
constexpr uint32_t ENV_SNAP_VERSION = 1;
struct EnvSnapHeader {
  char magic[8];
  uint32_t version, header_bytes;
  int64_t total_bytes;
  int32_t precision, num_envs, ring_depth, obs_dim;
  uint64_t hf_hash;            // FNV-1a of the height field's samples (0 on the plane)
  int32_t max_episode_steps;   // host field of the handle (b2q_set_max_episode_steps): restored by a load, not compared
  int32_t pad_;
  B2QConfig cfg;               // device, hf_host and max_episode_steps zeroed
};
#define B2Q_SNAP_FIELD(s, f, name) b2q_snap::Field{name, offsetof(s, f), sizeof(((s*)nullptr)->f)}
#define B2Q_SNAP_CFG(f) B2Q_SNAP_FIELD(EnvSnapHeader, cfg.f, #f)
// compared in this order by a load; the first difference is named in the error
const b2q_snap::Field ENV_SNAP_FIELDS[] = {
    B2Q_SNAP_FIELD(EnvSnapHeader, magic, "magic"), B2Q_SNAP_FIELD(EnvSnapHeader, version, "version"),
    B2Q_SNAP_FIELD(EnvSnapHeader, header_bytes, "header size"), B2Q_SNAP_FIELD(EnvSnapHeader, total_bytes, "size"),
    B2Q_SNAP_FIELD(EnvSnapHeader, precision, "precision"), B2Q_SNAP_FIELD(EnvSnapHeader, num_envs, "num_envs"),
    B2Q_SNAP_FIELD(EnvSnapHeader, ring_depth, "ring_depth"), B2Q_SNAP_FIELD(EnvSnapHeader, obs_dim, "obs_dim"),
    B2Q_SNAP_CFG(threads_per_block), B2Q_SNAP_CFG(sim_dt), B2Q_SNAP_CFG(action_repeat), B2Q_SNAP_CFG(solver_iters), B2Q_SNAP_CFG(erp),
    B2Q_SNAP_CFG(warmstart), B2Q_SNAP_CFG(contact_margin), B2Q_SNAP_CFG(action_interp), B2Q_SNAP_CFG(torque_limit), B2Q_SNAP_CFG(settle_steps),
    B2Q_SNAP_CFG(etg_enabled), B2Q_SNAP_CFG(action_filter), B2Q_SNAP_CFG(filter_highcut), B2Q_SNAP_CFG(etg_T), B2Q_SNAP_CFG(etg_T2),
    B2Q_SNAP_CFG(etg_sigma_sq), B2Q_SNAP_CFG(etg_amp), B2Q_SNAP_CFG(etg_phase0), B2Q_SNAP_CFG(etg_phase1), B2Q_SNAP_CFG(w_torso),
    B2Q_SNAP_CFG(w_feet), B2Q_SNAP_CFG(w_up), B2Q_SNAP_CFG(w_tau), B2Q_SNAP_CFG(w_stand), B2Q_SNAP_CFG(w_badfoot), B2Q_SNAP_CFG(w_footcontact),
    B2Q_SNAP_CFG(w_done), B2Q_SNAP_CFG(reward_p), B2Q_SNAP_CFG(vel_d), B2Q_SNAP_CFG(foot_radius), B2Q_SNAP_CFG(auto_reset),
    B2Q_SNAP_CFG(terrain_type), B2Q_SNAP_CFG(hf_nx), B2Q_SNAP_CFG(hf_ny), B2Q_SNAP_CFG(hf_x0), B2Q_SNAP_CFG(hf_y0), B2Q_SNAP_CFG(hf_cell),
    B2Q_SNAP_CFG(clip_motor_commands), B2Q_SNAP_CFG(max_angle_change), B2Q_SNAP_CFG(sensor_dis), B2Q_SNAP_CFG(sensor_contact),
    B2Q_SNAP_CFG(sensor_imu), B2Q_SNAP_CFG(sensor_motor), B2Q_SNAP_CFG(sensor_etg), B2Q_SNAP_CFG(obs_normal), B2Q_SNAP_CFG(noise_stdev),
    B2Q_SNAP_CFG(noise_seed), B2Q_SNAP_CFG(stuck_termination), B2Q_SNAP_CFG(body_collisions), B2Q_SNAP_CFG(motor_mode),
    B2Q_SNAP_CFG(joint_limits), B2Q_SNAP_CFG(external_force), B2Q_SNAP_CFG(base_damping), B2Q_SNAP_CFG(etg_foot_y_inset),
    B2Q_SNAP_CFG(knee_contacts), B2Q_SNAP_FIELD(EnvSnapHeader, hf_hash, "height field"),
};

struct EnvBase {
  B2QConfig cfg;
  int prec;
  std::string err;
  int64_t launches = 0;
  virtual ~EnvBase() {}
  virtual int set_dynamics(const uint8_t* mask, const void* dyn, cudaStream_t s) = 0;
  virtual int reset(const uint8_t* mask, const void* w, const void* b, const void* xoff, void* obs, cudaStream_t s) = 0;
  virtual int set_force(const void* f, cudaStream_t s) = 0;
  int obs_dim = B2Q_OBS_DIM;
  int act_dim() const { return cfg.motor_mode == 2 ? 5 * B2Q_ACT_DIM : B2Q_ACT_DIM; }   // HYBRID: a 5-tuple per motor
  virtual int step(const void* action, int donef, void* obs, void* rew, uint8_t* done, void* info, cudaStream_t s) = 0;
  virtual int step_host(const void* a, int donef, void* obs, void* rew, uint8_t* done, void* info, cudaStream_t s) = 0;
  virtual int get_state(void* out, cudaStream_t s) = 0;
  virtual int set_state(const void* in, cudaStream_t s) = 0;
  virtual int get_step_count(int32_t* out, cudaStream_t s) = 0;
  virtual void set_max_steps(int m) = 0;
  virtual int render(const void* state, const int32_t* env_ids, int V, const float* view, const float* proj, int W, int H, uint8_t* rgba, float* depth,
                     int32_t* seg, cudaStream_t s) = 0;
  virtual void view(EnvView* v) const = 0;
  virtual int64_t snapshot_bytes() const = 0;
  virtual int snapshot_save(void* dst, cudaStream_t s) = 0;
  virtual int snapshot_load(const void* src, cudaStream_t s) = 0;
  virtual int set_tiles(const double* tiles, int n_tiles, const int32_t* tile_of_env, cudaStream_t s) = 0;
};

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e_ = (call);                                                          \
    if (e_ != cudaSuccess) {                                                          \
      err = std::string(#call) + ": " + cudaGetErrorString(e_);                       \
      return B2Q_ECUDA;                                                               \
    }                                                                                 \
  } while (0)

template <typename T>
struct EnvT : EnvBase {
  Cfg<T> kc;
  Buffers<T> B;
  Model<T>* d_model = nullptr;
  T* d_def48 = nullptr;
  T* d_hf = nullptr;
  void* d_pool = nullptr;
  int tpb = 32;
  float hf_lo = 0.0f, hf_hi = 0.0f;

  ~EnvT() override {
    cudaSetDevice(cfg.device);
    if (d_pool) cudaFree(d_pool);
    if (d_model) cudaFree(d_model);
    if (d_def48) cudaFree(d_def48);
    if (d_hf) cudaFree(d_hf);
    if (d_tiles) cudaFree(d_tiles);
    if (tl.tile_of_env) cudaFree(const_cast<int32_t*>(tl.tile_of_env));
    if (st_act) cudaFree(st_act);
    if (h_flag) cudaFreeHost(h_flag);
    if (h_snap) cudaFreeHost(h_snap);
  }
  int grid_lanes() const { return (B.N * 4 + tpb - 1) / tpb; }

  int init(const B2QConfig& c) {
    cfg = c; prec = c.precision;
    tpb = c.threads_per_block ? c.threads_per_block : 32;
    if (const char* e = std::getenv("B2Q_HOST_IO")) host_io = std::atoi(e);   // 0: memcpy both ways, 1: zero-copy actions, 2: + zero-copy outputs
    CK(cudaSetDevice(c.device));
    int N = c.num_envs, Dm = c.ring_depth;
    if (c.terrain_type == 1) {
      size_t n = (size_t)c.hf_nx * c.hf_ny;
      T* tmp = (T*)malloc(n * sizeof(T));
      if (!tmp) { err = "host alloc failed"; return B2Q_ENOMEM; }
      for (size_t i = 0; i < n; i++) tmp[i] = (T)c.hf_host[i];
      hf_hash = b2q_snap::fnv1a(c.hf_host, n * sizeof(double));
      hf_lo = hf_hi = (float)tmp[0];   // height range of the field: the camera rays are clipped to it (b2q_render)
      for (size_t i = 0; i < n; i++) { hf_lo = std::fmin(hf_lo, (float)tmp[i]); hf_hi = std::fmax(hf_hi, (float)tmp[i]); }
      cudaError_t e1 = cudaMalloc(&d_hf, n * sizeof(T));
      if (e1 == cudaSuccess) e1 = cudaMemcpy(d_hf, tmp, n * sizeof(T), cudaMemcpyHostToDevice);
      free(tmp);
      CK(e1);
    }
    kc = make_cfg<T>(c, d_hf);
    Model<T> hm; build_model_host(hm, c.foot_radius, c.etg_T, c.etg_amp, c.etg_phase0, c.etg_phase1, c.etg_foot_y_inset);
    build_obs_map(hm, c); obs_dim = hm.obs_dim;
    feat = config_feat(c);
    if (feat) tpb = 32;   // the FEAT variant keeps a 36x36 solver scratch per robot in shared memory: one warp (8 robots) per CTA
    if (smem_bytes() > 48 * 1024) {   // opt-in dynamic shared memory above 48 KB (FEAT scratch, or the exchange areas of a 128-thread CTA)
      if (feat) {
        CK(cudaFuncSetAttribute(b2q_step_kernel<T, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
        CK(cudaFuncSetAttribute(b2q_settle_kernel<T, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
      } else {
        CK(cudaFuncSetAttribute(b2q_step_kernel<T, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
        CK(cudaFuncSetAttribute(b2q_settle_kernel<T, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
      }
    }
    CK(cudaHostAlloc((void**)&h_flag, sizeof(int), cudaHostAllocDefault));
    CK(cudaHostAlloc(&h_snap, b2q_snap::HDR_BYTES, cudaHostAllocDefault));
    CK(cudaMalloc((void**)&d_model, (sizeof(Model<T>) + 15) / 16 * 16));      // padded: the kernels stage it with 16-byte loads
    CK(cudaMemset(d_model, 0, (sizeof(Model<T>) + 15) / 16 * 16));
    CK(cudaMemcpy(d_model, &hm, sizeof(Model<T>), cudaMemcpyHostToDevice));
    double d48[48]; default_dyn_row(d48); T t48[48]; for (int i = 0; i < 48; i++) t48[i] = (T)d48[i];
    CK(cudaMalloc(&d_def48, sizeof(t48)));
    CK(cudaMemcpy(d_def48, t48, sizeof(t48), cudaMemcpyHostToDevice));
    // one pool for the SoA env state: [state NS | snap NS | snap_obs 12 | param NP | etg NE | ring Dm*24] packs x N, + step counters
    size_t packs = (size_t)(NS + NS + 12 + NP + NE + Dm * 24 + STUCK_H + 1) * N;
    size_t bytes = packs * sizeof(P4<T>) + (size_t)(N + 1) * sizeof(int);
    pool_bytes = bytes;
    CK(cudaMalloc(&d_pool, bytes));
    CK(cudaMemset(d_pool, 0, bytes));
    P4<T>* p = (P4<T>*)d_pool;
    B.N = N; B.Dm = Dm;
    B.state = p; p += (size_t)NS * N; B.snap = p; p += (size_t)NS * N; B.snap_obs = p; p += (size_t)12 * N;
    B.param = p; p += (size_t)NP * N; B.etg = p; p += (size_t)NE * N; B.ring = p; p += (size_t)Dm * 24 * N;
    B.pos_hist = p; p += (size_t)STUCK_H * N; B.extf = p; p += (size_t)N;
    B.step_count = (int*)p; d_flag = B.step_count + N;
    int rc = set_dynamics(nullptr, nullptr, 0);
    if (rc) return rc;
    rc = reset(nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    if (rc) return rc;
    CK(cudaDeviceSynchronize());
    return B2Q_OK;
  }
  size_t smem_bytes() const {   // model | obs stage | info stage | per-robot solver scratch
    return ((sizeof(Model<T>) + 31) & ~size_t(31)) + (size_t)(tpb / 4) * (OBS_DIM + INFO_DIM + scratch_floats(feat)) * sizeof(T);
  }

  int set_dynamics(const uint8_t* mask, const void* dyn, cudaStream_t s) override {
    CK(cudaSetDevice(cfg.device));
    int N = B.N;
    // latencies the two-sample-per-step observation ring can serve: n_lag <= ring_depth*R - 2 substeps (step_lane)
    const double max_lat = ((double)B.Dm * cfg.action_repeat - 2) * cfg.sim_dt * (1.0 + 1e-9);
    CK(cudaMemsetAsync(d_flag, 0, sizeof(int), s));
    b2q_pack_param_kernel<T><<<(N + 127) / 128, 128, 0, s>>>((const T*)dyn, d_def48, const_cast<P4<T>*>(B.param), mask, N, (T)max_lat, d_flag);
    CK(cudaMemcpyAsync(h_flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));      // set_dynamics is a rare, heavyweight call (it re-settles 500 substeps): one sync is fine
    launches += 1;
    if (*h_flag) {
      char buf[200];
      snprintf(buf, sizeof buf, "b2q_set_dynamics: a control_latency exceeds %.4f s, the most ring_depth=%d can serve (need ring_depth >= ceil((latency/sim_dt + 2) / action_repeat))", max_lat, B.Dm);
      err = buf;
      return B2Q_EINVAL;
    }
    return settle(mask, s);
  }
  int settle(const uint8_t* mask, cudaStream_t s) {
    if (n_tiles && feat) b2q_settle_tiles_kernel<T, 1><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, tl, d_model, B, mask);
    else if (n_tiles) b2q_settle_tiles_kernel<T, 0><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, tl, d_model, B, mask);
    else if (feat) b2q_settle_kernel<T, 1><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, d_model, B, mask);
    else b2q_settle_kernel<T, 0><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, d_model, B, mask);
    launches += 1;
    CK(cudaGetLastError());
    return B2Q_OK;
  }
  int reset(const uint8_t* mask, const void* w, const void* b, const void* xoff, void* obs, cudaStream_t s) override {
    CK(cudaSetDevice(cfg.device));
    int N = B.N;
    if (w || b) { b2q_pack_etg_kernel<T><<<(N + 127) / 128, 128, 0, s>>>((const T*)w, (const T*)b, const_cast<P4<T>*>(B.etg), mask, N); launches++; }
    const size_t smem_reset = ((sizeof(Model<T>) + 31) & ~size_t(31)) + (size_t)(tpb / 4) * OBS_DIM * sizeof(T);   // model + observation stage only
    b2q_reset_kernel<T><<<grid_lanes(), tpb, smem_reset, s>>>(kc, d_model, B, mask, (const T*)xoff, (T*)obs);
    launches++;
    CK(cudaGetLastError());
    return B2Q_OK;
  }
  int set_force(const void* f, cudaStream_t s) override {
    if (!cfg.external_force) { err = "b2q_set_external_force: the handle was created with external_force = 0"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    b2q_pack_force_kernel<T><<<(B.N + 127) / 128, 128, 0, s>>>((const T*)f, const_cast<P4<T>*>(B.extf), B.N);
    launches++;
    CK(cudaGetLastError());
    return B2Q_OK;
  }
  int feat = 0; int* d_flag = nullptr; int* h_flag = nullptr;
  int step(const void* action, int donef, void* obs, void* rew, uint8_t* done, void* info, cudaStream_t s) override {
    if (!action || !obs || !rew || !done || !info) { err = "b2q_step: null device pointer"; return B2Q_EINVAL; }
    { int cur = -1; if (cudaGetDevice(&cur) != cudaSuccess || cur != cfg.device) CK(cudaSetDevice(cfg.device)); }   // handles are per GPU
    if (n_tiles && feat)
      b2q_step_tiles_kernel<T, 1><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, tl, d_model, B, (const T*)action, donef, cfg.auto_reset, (T*)obs, (T*)rew, done, (T*)info);
    else if (n_tiles)
      b2q_step_tiles_kernel<T, 0><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, tl, d_model, B, (const T*)action, donef, cfg.auto_reset, (T*)obs, (T*)rew, done, (T*)info);
    else if (feat) b2q_step_kernel<T, 1><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, d_model, B, (const T*)action, donef, cfg.auto_reset, (T*)obs, (T*)rew, done, (T*)info);
    else b2q_step_kernel<T, 0><<<grid_lanes(), tpb, smem_bytes(), s>>>(kc, d_model, B, (const T*)action, donef, cfg.auto_reset, (T*)obs, (T*)rew, done, (T*)info);
    launches++;
    CK(cudaGetLastError());
    return B2Q_OK;
  }
  // device staging for the host-buffer API (allocated on first use)
  T* st_act = nullptr; T* st_obs = nullptr; T* st_rew = nullptr; uint8_t* st_done = nullptr; T* st_info = nullptr;
  int step_host(const void* a, int donef, void* obs, void* rew, uint8_t* done, void* info, cudaStream_t s) override {
    if (!a || !obs || !rew || !done) { err = "b2q_step_host: null host pointer"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    const size_t N = (size_t)B.N;
    if (!st_act) {
      size_t bytes = N * ((size_t)act_dim() + OBS_DIM + 1 + INFO_DIM) * sizeof(T) + N + 512;
      void* p = nullptr;
      CK(cudaMalloc(&p, bytes));
      // layout: act | obs | rew | done (bytes) | pad | info  — obs/rew/done contiguous so one D2H can serve all three
      st_act = (T*)p; st_obs = st_act + N * (size_t)act_dim(); st_rew = st_obs + N * OBS_DIM; st_done = (uint8_t*)(st_rew + N);
      st_info = (T*)((uint8_t*)p + ((N * ((size_t)act_dim() + OBS_DIM + 1) * sizeof(T) + N + 255) / 256) * 256);
    }
    // Pinned (page-locked) host buffers are device-addressable under unified addressing: the kernel then reads the actions
    // straight from host memory (one coalesced 12-float row per robot, read once) instead of waiting for a separate H2D copy,
    // and — host_io >= 2 — stores its staged, coalesced observation block plus reward/done straight to host memory.
    // Pageable buffers, and the scattered info rows, go through the device staging area and cudaMemcpyAsync.
    const T* act_dev = st_act;
    if (host_io >= 1 && (act_dev = (const T*)mapped(a)) == nullptr) act_dev = st_act;
    if (act_dev == st_act) CK(cudaMemcpyAsync(st_act, a, N * (size_t)act_dim() * sizeof(T), cudaMemcpyHostToDevice, s));
    T* obs_dev = nullptr; T* rew_dev = nullptr; uint8_t* done_dev = nullptr;
    if (host_io >= 2) { obs_dev = (T*)mapped(obs); rew_dev = (T*)mapped(rew); done_dev = (uint8_t*)mapped(done); }
    const bool direct = obs_dev && rew_dev && done_dev;
    // info rows are staged in shared memory and stored as one coalesced block per CTA like the observations: zero-copy too
    T* info_dev = (direct && info) ? (T*)mapped(info) : nullptr;
    int rc = direct ? step(act_dev, donef, obs_dev, rew_dev, done_dev, info_dev ? info_dev : st_info, s) : step(act_dev, donef, st_obs, st_rew, st_done, st_info, s);
    if (rc) return rc;
    if (info_dev) info = nullptr;
    const size_t b_obs = N * (size_t)obs_dim * sizeof(T), b_rew = N * sizeof(T);
    if (direct) {
    } else if ((uint8_t*)rew == (uint8_t*)obs + b_obs && done == (uint8_t*)rew + b_rew) {
      CK(cudaMemcpyAsync(obs, st_obs, b_obs + b_rew + N, cudaMemcpyDeviceToHost, s));      // caller's host buffers are contiguous too
    } else {
      CK(cudaMemcpyAsync(obs, st_obs, b_obs, cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(rew, st_rew, b_rew, cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(done, st_done, N, cudaMemcpyDeviceToHost, s));
    }
    if (info) CK(cudaMemcpyAsync(info, st_info, N * INFO_DIM * sizeof(T), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return B2Q_OK;
  }
  // device alias of a pinned host pointer (nullptr for pageable memory); queried every call — a cached answer could go
  // stale if the caller frees the pinned block and the address is reused by pageable memory
  int host_io = 2;
  void* mapped(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) return at.devicePointer;
    cudaGetLastError();
    return nullptr;
  }
  int get_state(void* out, cudaStream_t s) override {
    if (!out) { err = "b2q_get_state: null pointer"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    b2q_get_state_kernel<T><<<(B.N + 127) / 128, 128, 0, s>>>(B.state, (T*)out, B.N); launches++;
    CK(cudaGetLastError());
    return B2Q_OK;
  }
  int set_state(const void* in, cudaStream_t s) override {
    if (!in) { err = "b2q_set_state: null pointer"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    b2q_set_state_kernel<T><<<(B.N + 127) / 128, 128, 0, s>>>(B.state, (const T*)in, B.N); launches++;
    CK(cudaGetLastError());
    return B2Q_OK;
  }
  int get_step_count(int32_t* out, cudaStream_t s) override {
    if (!out) { err = "b2q_get_step_count: null pointer"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    CK(cudaMemcpyAsync(out, B.step_count, sizeof(int) * B.N, cudaMemcpyDeviceToDevice, s));
    return B2Q_OK;
  }
  void set_max_steps(int m) override { cfg.max_episode_steps = m; kc.max_steps = m; }   // kc goes to the step kernel by value
  // The pool is the whole device state a step or reset reads and writes (the model, default dynamics and height field are fixed at
  // create); cfg.max_episode_steps (= kc.max_steps) is the one host field that changes after create.  `launches` only counts.
  size_t pool_bytes = 0;
  uint64_t hf_hash = 0;
  void* h_snap = nullptr;   // pinned landing slot of a loaded header
  int64_t snapshot_bytes() const override { return (int64_t)(b2q_snap::HDR_BYTES + pool_bytes); }
  EnvSnapHeader snap_header() const {
    EnvSnapHeader h;
    std::memset(&h, 0, sizeof h);
    std::memcpy(h.magic, "B2QENV\0\0", 8);
    h.version = ENV_SNAP_VERSION; h.header_bytes = (uint32_t)b2q_snap::HDR_BYTES; h.total_bytes = snapshot_bytes();
    h.precision = prec; h.num_envs = B.N; h.ring_depth = B.Dm; h.obs_dim = obs_dim; h.hf_hash = hf_hash; h.max_episode_steps = cfg.max_episode_steps;
    h.cfg = cfg; h.cfg.device = 0; h.cfg.hf_host = nullptr; h.cfg.max_episode_steps = 0;
    return h;
  }
  int snapshot_save(void* dst, cudaStream_t s) override {
    if (n_tiles) { err = "b2q_snapshot_save: not on a terrain-atlas handle (the snapshot header hashes one height field)"; return B2Q_EINVAL; }
    if (!dst || ((size_t)dst & 15)) { err = "b2q_snapshot_save: dst must be a 16-byte aligned device pointer"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    CK(b2q_snap::write_header(snap_header(), dst, s));
    CK(cudaMemcpyAsync((char*)dst + b2q_snap::HDR_BYTES, d_pool, pool_bytes, cudaMemcpyDeviceToDevice, s));
    launches++;
    return B2Q_OK;
  }
  int snapshot_load(const void* src, cudaStream_t s) override {
    if (n_tiles) { err = "b2q_snapshot_load: not on a terrain-atlas handle (the snapshot header hashes one height field)"; return B2Q_EINVAL; }
    if (!src || ((size_t)src & 15)) { err = "b2q_snapshot_load: src must be a 16-byte aligned device pointer"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    // the refusal is a return code, so the header has to reach the host first: one small copy, waited for
    CK(cudaMemcpyAsync(h_snap, src, sizeof(EnvSnapHeader), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const EnvSnapHeader mine = snap_header();
    if (const char* f = b2q_snap::first_difference(h_snap, &mine, ENV_SNAP_FIELDS, (int)(sizeof ENV_SNAP_FIELDS / sizeof ENV_SNAP_FIELDS[0]))) {
      err = std::string("b2q_snapshot_load: the blob's ") + f + " differs from this handle's";
      return B2Q_EINVAL;
    }
    const int m = static_cast<const EnvSnapHeader*>(h_snap)->max_episode_steps;
    if (m < 0) { err = "b2q_snapshot_load: the blob's max_episode_steps is negative"; return B2Q_EINVAL; }
    CK(cudaMemcpyAsync(d_pool, (const char*)src + b2q_snap::HDR_BYTES, pool_bytes, cudaMemcpyDeviceToDevice, s));
    set_max_steps(m);
    return B2Q_OK;
  }
  void view(EnvView* v) const override {
    v->N = B.N; v->obs_dim = obs_dim; v->elem_size = (int)sizeof(T); v->device = cfg.device; v->etg_enabled = cfg.etg_enabled;
    v->step_count = B.step_count; v->model = d_model; v->state = B.state;
  }
  int render(const void* state, const int32_t* env_ids, int V, const float* view, const float* proj, int W, int H, uint8_t* rgba, float* depth,
             int32_t* seg, cudaStream_t s) override {
    if (n_tiles) { err = "b2q_render: not on a terrain-atlas handle (the renderer ray-casts the handle's one height field)"; return B2Q_EINVAL; }
    if (!state || !env_ids || !view || !proj) { err = "b2q_render: null state, env_ids, view or proj"; return B2Q_EINVAL; }
    if (V < 1 || V > 65535) { err = "b2q_render: V must be in [1, 65535]"; return B2Q_EINVAL; }
    if (W < 1 || H < 1 || W > 16384 || H > 16384) { err = "b2q_render: width and height must be in [1, 16384]"; return B2Q_EINVAL; }
    if ((size_t)rgba & 3) { err = "b2q_render: rgba must be 4-byte aligned"; return B2Q_EINVAL; }
    CK(cudaSetDevice(cfg.device));
    RenderArgs<T> a;
    build_model_host(a.md, cfg.foot_radius, cfg.etg_T, cfg.etg_amp, cfg.etg_phase0, cfg.etg_phase1, cfg.etg_foot_y_inset);
    a.tr.type = kc.terrain; a.tr.nx = kc.hf_nx; a.tr.ny = kc.hf_ny;
    a.tr.x0 = (float)cfg.hf_x0; a.tr.y0 = (float)cfg.hf_y0; a.tr.icell = (float)kc.hf_icell; a.tr.lo = hf_lo; a.tr.hi = hf_hi;
    a.hf = d_hf; a.state = (const T*)state; a.N = B.N; a.env_ids = env_ids; a.view = view; a.proj = proj;
    a.W = W; a.H = H; a.rgba = rgba; a.depth = depth; a.seg = seg;
    CK(render_launch<T>(a, V, s));
    launches++;
    return B2Q_OK;
  }
  // terrain atlas: n_tiles > 0 once b2q_set_terrain_tiles succeeded; kc.hf then points at d_tiles
  T* d_tiles = nullptr;
  Tiles tl{nullptr, 0};
  int n_tiles = 0;
  int set_tiles(const double* tiles, int nt, const int32_t* tile_of_env, cudaStream_t s) override {
    if (cfg.terrain_type != 1) { err = "b2q_set_terrain_tiles: needs a height-field handle (terrain_type 1): its hf_* fields give the tiles' grid"; return B2Q_EINVAL; }
    if (!tiles || !tile_of_env) { err = "b2q_set_terrain_tiles: null tiles or tile_of_env"; return B2Q_EINVAL; }
    if (nt < 1) { err = "b2q_set_terrain_tiles: n_tiles must be >= 1"; return B2Q_EINVAL; }
    for (int i = 0; i < B.N; i++) {
      if (tile_of_env[i] < 0 || tile_of_env[i] >= nt) {
        char buf[160];
        snprintf(buf, sizeof buf, "b2q_set_terrain_tiles: tile_of_env[%d] = %d is outside [0, %d)", i, (int)tile_of_env[i], nt);
        err = buf;
        return B2Q_EINVAL;
      }
    }
    CK(cudaSetDevice(cfg.device));
    const size_t per = (size_t)cfg.hf_nx * cfg.hf_ny, n = per * (size_t)nt;   // the kernels offset by tile * per in 64 bits
    T* tmp = (T*)malloc(n * sizeof(T));
    if (!tmp) { err = "b2q_set_terrain_tiles: host alloc failed"; return B2Q_ENOMEM; }
    for (size_t i = 0; i < n; i++) tmp[i] = (T)tiles[i];
    CK(cudaStreamSynchronize(s));   // the previous atlas may still be read by launches on the stream
    if (d_tiles) { cudaFree(d_tiles); d_tiles = nullptr; }
    if (tl.tile_of_env) { cudaFree(const_cast<int32_t*>(tl.tile_of_env)); tl.tile_of_env = nullptr; }
    n_tiles = 0; kc.hf = d_hf;
    int32_t* d_map = nullptr;
    cudaError_t e1 = cudaMalloc(&d_tiles, n * sizeof(T));
    if (e1 == cudaSuccess) e1 = cudaMemcpy(d_tiles, tmp, n * sizeof(T), cudaMemcpyHostToDevice);
    free(tmp);
    if (e1 == cudaSuccess) e1 = cudaMalloc(&d_map, (size_t)B.N * sizeof(int32_t));
    if (e1 == cudaSuccess) e1 = cudaMemcpy(d_map, tile_of_env, (size_t)B.N * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e1 != cudaSuccess) {
      if (d_tiles) cudaFree(d_tiles);
      if (d_map) cudaFree(d_map);
      d_tiles = nullptr;
      CK(e1);
    }
    if (smem_bytes() > 48 * 1024) {
      if (feat) {
        CK(cudaFuncSetAttribute(b2q_step_tiles_kernel<T, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
        CK(cudaFuncSetAttribute(b2q_settle_tiles_kernel<T, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
      } else {
        CK(cudaFuncSetAttribute(b2q_step_tiles_kernel<T, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
        CK(cudaFuncSetAttribute(b2q_settle_tiles_kernel<T, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
      }
    }
    tl.tile_of_env = d_map; tl.tile_elems = (long long)per;
    n_tiles = nt; kc.hf = d_tiles;
    return settle(nullptr, s);   // every env's reset snapshot, settled on its own tile with the dynamics it has
  }
};

}  // namespace

struct B2QEnv { EnvBase* impl; };

namespace b2q {
int env_view(B2QHandle h, EnvView* v) {
  if (!h || !v) return B2Q_EINVAL;
  h->impl->view(v);
  return B2Q_OK;
}
void env_set_error(B2QHandle h, const char* msg) { if (h) h->impl->err = msg; }
}  // namespace b2q

extern "C" {

void b2q_default_config(B2QConfig* cfg) { if (cfg) default_config(cfg); }
const char* b2q_version(void) { return "b2q 0.1.0 (sm_90a)"; }

int b2q_create(const B2QConfig* cfg, B2QHandle* out) {
  if (!cfg || !out) { g_create_err = "null argument"; return B2Q_EINVAL; }
  *out = nullptr;
  if (const char* m = validate_config(*cfg)) { g_create_err = m; return B2Q_EINVAL; }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) { g_create_err = std::string("no CUDA device (no CPU fallback exists): ") + cudaGetErrorString(e); return B2Q_ECUDA; }
  if (cfg->device < 0 || cfg->device >= ndev) { g_create_err = "device ordinal out of range"; return B2Q_EINVAL; }
  EnvBase* impl = nullptr;
  int rc;
  if (cfg->precision == 0) { auto* t = new (std::nothrow) EnvT<float>(); if (!t) return B2Q_ENOMEM; rc = t->init(*cfg); impl = t; }
  else { auto* t = new (std::nothrow) EnvT<double>(); if (!t) return B2Q_ENOMEM; rc = t->init(*cfg); impl = t; }
  if (rc != B2Q_OK) { g_create_err = impl->err; delete impl; return rc; }
  B2QEnv* h = new (std::nothrow) B2QEnv{impl};
  if (!h) { delete impl; return B2Q_ENOMEM; }
  *out = h;
  return B2Q_OK;
}
int b2q_destroy(B2QHandle h) { if (!h) return B2Q_EINVAL; delete h->impl; delete h; return B2Q_OK; }
const char* b2q_last_error(B2QHandle h) { return h ? h->impl->err.c_str() : g_create_err.c_str(); }
int b2q_num_envs(B2QHandle h) { return h ? h->impl->cfg.num_envs : B2Q_EINVAL; }
int b2q_obs_dim(B2QHandle h) { return h ? h->impl->obs_dim : B2Q_EINVAL; }
int b2q_act_dim(B2QHandle h) { return h ? h->impl->act_dim() : B2Q_EINVAL; }
int b2q_info_dim(B2QHandle h) { return h ? B2Q_INFO_DIM : B2Q_EINVAL; }
int b2q_elem_size(B2QHandle h) { return h ? (h->impl->prec ? 8 : 4) : B2Q_EINVAL; }
int b2q_set_dynamics(B2QHandle h, const uint8_t* m, const void* dyn, void* s) { return h ? h->impl->set_dynamics(m, dyn, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_reset(B2QHandle h, const uint8_t* m, const void* w, const void* b, void* obs, void* s) { return h ? h->impl->reset(m, w, b, nullptr, obs, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_reset_ex(B2QHandle h, const uint8_t* m, const void* w, const void* b, const void* xoff, void* obs, void* s) {
  return h ? h->impl->reset(m, w, b, xoff, obs, (cudaStream_t)s) : B2Q_EINVAL;
}
int b2q_set_external_force(B2QHandle h, const void* f, void* s) { return h ? h->impl->set_force(f, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_step(B2QHandle h, const void* a, int donef, void* obs, void* rew, uint8_t* done, void* info, void* s) {
  return h ? h->impl->step(a, donef, obs, rew, done, info, (cudaStream_t)s) : B2Q_EINVAL;
}
int b2q_step_host(B2QHandle h, const void* a, int donef, void* obs, void* rew, uint8_t* done, void* info, void* s) {
  return h ? h->impl->step_host(a, donef, obs, rew, done, info, (cudaStream_t)s) : B2Q_EINVAL;
}
void* b2q_host_alloc(size_t bytes) { void* p = nullptr; return cudaHostAlloc(&p, bytes, cudaHostAllocDefault) == cudaSuccess ? p : nullptr; }
void b2q_host_free(void* p) { if (p) cudaFreeHost(p); }
int b2q_get_state(B2QHandle h, void* out, void* s) { return h ? h->impl->get_state(out, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_set_state(B2QHandle h, const void* in, void* s) { return h ? h->impl->set_state(in, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_get_step_count(B2QHandle h, int32_t* out, void* s) { return h ? h->impl->get_step_count(out, (cudaStream_t)s) : B2Q_EINVAL; }
int64_t b2q_launch_count(B2QHandle h) { return h ? h->impl->launches : 0; }
int b2q_set_max_episode_steps(B2QHandle h, int m) {
  if (!h || m < 0) return B2Q_EINVAL;
  h->impl->set_max_steps(m);
  return B2Q_OK;
}
int64_t b2q_snapshot_bytes(B2QHandle h) { return h ? h->impl->snapshot_bytes() : B2Q_EINVAL; }
int b2q_snapshot_save(B2QHandle h, void* dst, void* s) { return h ? h->impl->snapshot_save(dst, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_snapshot_load(B2QHandle h, const void* src, void* s) { return h ? h->impl->snapshot_load(src, (cudaStream_t)s) : B2Q_EINVAL; }
int b2q_set_terrain_tiles(B2QHandle h, const double* tiles_host, int n_tiles, const int32_t* tile_of_env, void* stream) {
  return h ? h->impl->set_tiles(tiles_host, n_tiles, tile_of_env, (cudaStream_t)stream) : B2Q_EINVAL;
}
int b2q_render(B2QHandle h, const void* state, const int32_t* env_ids, int V, const float* view, const float* proj, int width, int height, uint8_t* rgba,
               float* depth, int32_t* seg, void* stream) {
  return h ? h->impl->render(state, env_ids, V, view, proj, width, height, rgba, depth, seg, (cudaStream_t)stream) : B2Q_EINVAL;
}

#ifdef B2Q_REGION_CLOCKS
// Debug ABI of the region-clock build only (not in include/b2q.h, absent from the product library): waits for the device, copies the
// first n_warps rows of the step kernel's region clocks to `out` ([n_warps][12] u64: the RC_* regions of b2q_sim.cuh, entry-to-exit
// cycles, launches; may be NULL) and zeroes every row when `clear` is set.
int b2q_region_clocks(int device, uint64_t* out, int n_warps, int clear) {
  static_assert(RC_COLS == 12, "the row layout documented above");
  if (n_warps < 0 || n_warps > RC_MAX_WARPS) return B2Q_EINVAL;
  if (cudaSetDevice(device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return B2Q_ECUDA;
  const size_t bytes = (size_t)n_warps * RC_COLS * sizeof(unsigned long long);
  if (out && bytes && cudaMemcpyFromSymbol(out, g_region_clocks, bytes) != cudaSuccess) return B2Q_ECUDA;
  if (clear) {
    void* p = nullptr;
    if (cudaGetSymbolAddress(&p, g_region_clocks) != cudaSuccess || cudaMemset(p, 0, sizeof(g_region_clocks)) != cudaSuccess) return B2Q_ECUDA;
    if (cudaDeviceSynchronize() != cudaSuccess) return B2Q_ECUDA;
  }
  return B2Q_OK;
}
#endif

}  // extern "C"
