// b2q_rpm.cu — device replay memory kernels (include/b2q_rpm.h): batched ring append and uniform minibatch gather; the behaviour-cloning
// student observation (sensor noise + pair append) and the permutation gather on a device cursor.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include "../../include/b2q_rpm.h"
#include "b2q_philox.cuh"

namespace {
__global__ void rpm_append_kernel(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term, const float* obs, const float* act, const float* rew,
                                  const float* next_obs, const float* term, int n, int od, int ad, int pos, int cap) {
  int i = blockIdx.x, t = threadIdx.x;
  if (i >= n) return;
  size_t slot = (size_t)((pos + i) % cap);
  for (int k = t; k < od; k += blockDim.x) { s_obs[slot * od + k] = obs[(size_t)i * od + k]; s_next[slot * od + k] = next_obs[(size_t)i * od + k]; }
  for (int k = t; k < ad; k += blockDim.x) s_act[slot * ad + k] = act[(size_t)i * ad + k];
  if (t == 0) { s_rew[slot] = rew[i]; s_term[slot] = term[i]; }
}
__device__ __forceinline__ uint32_t mix(uint64_t x) {  // splitmix64 finaliser
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; x ^= x >> 31;
  return (uint32_t)(x >> 32);
}
__global__ void rpm_sample_kernel(const float* s_obs, const float* s_act, const float* s_rew, const float* s_next, const float* s_term, float* obs, float* act,
                                  float* rew, float* next_obs, float* term, int batch, int od, int ad, int size, uint64_t seed) {
  int i = blockIdx.x, t = threadIdx.x;
  if (i >= batch) return;
  size_t slot = (size_t)(((uint64_t)mix(seed * 0x100000001B3ull + (uint64_t)i) * (uint64_t)size) >> 32);   // uniform in [0,size)
  for (int k = t; k < od; k += blockDim.x) { obs[(size_t)i * od + k] = s_obs[slot * od + k]; next_obs[(size_t)i * od + k] = s_next[slot * od + k]; }
  for (int k = t; k < ad; k += blockDim.x) act[(size_t)i * ad + k] = s_act[slot * ad + k];
  if (t == 0) { rew[i] = s_rew[slot]; term[i] = s_term[slot]; }
}
// ---- device-side cursor: state = {ring position, fill level, sample counter} lives in device memory, so that append / sample can be captured
//      once in a CUDA graph (kernel arguments frozen) and replayed every iteration
__global__ void rpm_append_cursor_kernel(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term, const float* obs, const float* act, const float* rew,
                                         const float* next_obs, const float* term, int n, int od, int ad, int cap, const long long* state) {
  int i = blockIdx.x, t = threadIdx.x;
  if (i >= n) return;
  size_t slot = (size_t)((state[0] + i) % cap);
  for (int k = t; k < od; k += blockDim.x) { s_obs[slot * od + k] = obs[(size_t)i * od + k]; s_next[slot * od + k] = next_obs[(size_t)i * od + k]; }
  for (int k = t; k < ad; k += blockDim.x) s_act[slot * ad + k] = act[(size_t)i * ad + k];
  if (t == 0) { s_rew[slot] = rew[i]; s_term[slot] = term[i]; }
}
__global__ void rpm_advance_kernel(long long* state, int n, int cap) { state[0] = (state[0] + n) % cap; state[1] = state[1] + n < cap ? state[1] + n : cap; }
__global__ void rpm_sample_cursor_kernel(const float* s_obs, const float* s_act, const float* s_rew, const float* s_next, const float* s_term, float* obs, float* act,
                                         float* rew, float* next_obs, float* term, int batch, int od, int ad, uint64_t seed, const long long* state) {
  int i = blockIdx.x, t = threadIdx.x;
  if (i >= batch) return;
  const uint64_t size = (uint64_t)state[1], sd = seed + (uint64_t)state[2];
  size_t slot = (size_t)(((uint64_t)mix(sd * 0x100000001B3ull + (uint64_t)i) * size) >> 32);
  for (int k = t; k < od; k += blockDim.x) { obs[(size_t)i * od + k] = s_obs[slot * od + k]; next_obs[(size_t)i * od + k] = s_next[slot * od + k]; }
  for (int k = t; k < ad; k += blockDim.x) act[(size_t)i * ad + k] = s_act[slot * ad + k];
  if (t == 0) { rew[i] = s_rew[slot]; term[i] = s_term[slot]; }
}
__global__ void rpm_count_kernel(long long* state) { state[2] += 1; }

// ---- masked append on the device cursor: row i goes to slot (state[0] + rank_i) % cap, rank_i = number of valid rows before i.  The call has
//      no scratch memory, so each CTA recounts the mask before its tile (word loads); the grid is capped at MASK_MAX_CTAS so that this recount
//      costs at most MASK_MAX_CTAS * n bytes of (L2-resident) reads.  The count of valid rows never leaves the device.
constexpr int MASK_THREADS = 256, MASK_MAX_CTAS = 512;
__device__ __forceinline__ int count_valid(const uint8_t* __restrict__ v, int end) {   // nonzero bytes of v[0, end) seen by this thread
  int c = 0;
  const int head = min(end, (int)((4 - ((uintptr_t)v & 3)) & 3));
  for (int j = threadIdx.x; j < head; j += blockDim.x) c += v[j] != 0;
  const uint32_t* w = (const uint32_t*)(v + head);
  const int nw = (end - head) >> 2;
  for (int j = threadIdx.x; j < nw; j += blockDim.x) c += __popc(__vcmpne4(__ldg(w + j), 0u)) >> 3;
  for (int j = head + 4 * nw + threadIdx.x; j < end; j += blockDim.x) c += v[j] != 0;
  return c;
}
__device__ __forceinline__ int block_sum(int x, int* red) {     // every thread gets the CTA's sum; red = 32 ints of shared memory
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  int s = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += red[w];
  return s;
}
__global__ void __launch_bounds__(MASK_THREADS) rpm_append_masked_kernel(float* __restrict__ s_obs, float* __restrict__ s_act, float* __restrict__ s_rew,
    float* __restrict__ s_next, float* __restrict__ s_term, const float* __restrict__ obs, const float* __restrict__ act, const float* __restrict__ rew,
    const float* __restrict__ next_obs, const float* __restrict__ term, const uint8_t* __restrict__ valid, int n, int od, int ad, int cap, int tile,
    const long long* __restrict__ state) {
  __shared__ int red[32], rows[MASK_THREADS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = MASK_THREADS / 32;
  const int lo = blockIdx.x * tile, hi = min(lo + tile, n);
  long long base = state[0] + block_sum(count_valid(valid, lo), red);          // ring slot of this tile's first valid row (before the wrap)
  for (int c0 = lo; c0 < hi; c0 += MASK_THREADS) {                                // chunks of 256 rows: ballot scan, compacted row list, warp per row
    const int i = c0 + (int)threadIdx.x;
    const bool f = i < hi && valid[i] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    __syncthreads();                                                              // the previous chunk's copy has finished reading rows[]
    if (lane == 0) red[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < nwarps; w++) { before += w < warp ? red[w] : 0; total += red[w]; }
    if (f) rows[before + __popc(bal & ((1u << lane) - 1u))] = i;
    __syncthreads();
    for (int r = warp; r < total; r += nwarps) {
      const size_t src = (size_t)rows[r], slot = (size_t)((base + r) % cap);
      for (int k = lane; k < od; k += 32) { s_obs[slot * od + k] = obs[src * od + k]; s_next[slot * od + k] = next_obs[src * od + k]; }
      for (int k = lane; k < ad; k += 32) s_act[slot * ad + k] = act[src * ad + k];
      if (lane == 0) { s_rew[slot] = rew[src]; s_term[slot] = term[src]; }
    }
    base += total;
  }
}
// one CTA, after the copy (stream order): advance position and fill level by the number of valid rows; the sample counter stays
__global__ void __launch_bounds__(MASK_THREADS) rpm_advance_masked_kernel(long long* state, const uint8_t* __restrict__ valid, int n, int cap) {
  __shared__ int red[32];
  const int m = block_sum(count_valid(valid, n), red);
  if (threadIdx.x == 0) { state[0] = (state[0] + m) % cap; state[1] = state[1] + m < cap ? state[1] + m : cap; }
}

// ---- behaviour cloning: student observation with sensor noise (+ optional ring append), and the permutation gather on a device cursor
constexpr int BC_THREADS = 256;
__device__ __forceinline__ float bc_sigma(int c) {      // BCtrain.py:55-58 over the sensor normalisers (bc.NOISE); 0 = no noise on column c
  return c < 7 ? 0.f : c < 10 ? 0.6f : c < 13 ? 0.2f : c < 25 ? 0.1f : c < 37 ? 0.5f : 0.f;
}
// one thread per element of obs [n, D]: coalesced reads of the expert rows, coalesced writes of both ring rows and the student row
__global__ void __launch_bounds__(BC_THREADS) bc_observe_kernel(const float* __restrict__ obs, int n, int D, float* __restrict__ student,
    float* __restrict__ ring_obs, float* __restrict__ ring_ref, int pos, int cap, uint64_t key, int noise) {
  const size_t total = (size_t)n * D;
  for (size_t e = (size_t)blockIdx.x * BC_THREADS + threadIdx.x; e < total; e += (size_t)gridDim.x * BC_THREADS) {
    const int i = (int)(e / D), c = (int)(e - (size_t)i * D);
    const float o = obs[e];
    const size_t slot = ring_ref ? (size_t)(((long long)pos + i) % cap) : 0;
    if (ring_ref) ring_ref[slot * D + c] = o;
    if (c < 3) continue;
    const float sig = noise ? bc_sigma(c) : 0.f;
    const float v = sig != 0.f ? __fadd_rn(o, __fmul_rn(sig, b2q_philox::philox_normal(key, (uint32_t)i, (uint32_t)c))) : o;
    student[(size_t)i * (D - 3) + c - 3] = v;
    if (ring_obs) ring_obs[slot * (D - 3) + c - 3] = v;
  }
}
// one thread per element of the [batch, od + rd] gathered pair; state[0] is the pass offset
__global__ void __launch_bounds__(BC_THREADS) bc_gather_kernel(const float* __restrict__ ring_obs, const float* __restrict__ ring_ref,
    const int64_t* __restrict__ perm, int perm_len, const long long* __restrict__ state, float* __restrict__ out_obs, float* __restrict__ out_ref,
    int batch, int od, int rd) {
  const int w = od + rd;
  const long long off = state[0];
  for (int e = blockIdx.x * BC_THREADS + threadIdx.x; e < batch * w; e += gridDim.x * BC_THREADS) {
    const int r = e / w, c = e - r * w;
    if (off + r >= perm_len) continue;
    const size_t src = (size_t)perm[off + r];
    if (c < od) out_obs[(size_t)r * od + c] = ring_obs[src * od + c];
    else out_ref[(size_t)r * rd + c - od] = ring_ref[src * rd + c - od];
  }
}
__global__ void bc_cursor_advance_kernel(long long* state, int batch) { state[0] += batch; }
}  // namespace

extern "C" {
int b2q_rpm_append(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term, const float* obs, const float* act, const float* rew,
                   const float* next_obs, const float* term, const uint8_t* valid, int n, int od, int ad, int pos, int cap, void* stream) {
  (void)valid;
  if (!s_obs || !s_act || !s_rew || !s_next || !s_term || !obs || !act || !rew || !next_obs || !term || n < 1 || cap < n || pos < 0) return -1;
  rpm_append_kernel<<<n, 64, 0, (cudaStream_t)stream>>>(s_obs, s_act, s_rew, s_next, s_term, obs, act, rew, next_obs, term, n, od, ad, pos, cap);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_rpm_sample(const float* s_obs, const float* s_act, const float* s_rew, const float* s_next, const float* s_term, float* obs, float* act, float* rew,
                   float* next_obs, float* term, int batch, int od, int ad, int size, uint64_t seed, void* stream) {
  if (!s_obs || !obs || batch < 1 || size < 1) return -1;
  rpm_sample_kernel<<<batch, 64, 0, (cudaStream_t)stream>>>(s_obs, s_act, s_rew, s_next, s_term, obs, act, rew, next_obs, term, batch, od, ad, size, seed);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_rpm_append_cursor(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term, const float* obs, const float* act, const float* rew,
                          const float* next_obs, const float* term, int n, int od, int ad, int cap, long long* state, void* stream) {
  if (!s_obs || !s_act || !s_rew || !s_next || !s_term || !obs || !act || !rew || !next_obs || !term || !state || n < 1 || cap < n) return -1;
  rpm_append_cursor_kernel<<<n, 64, 0, (cudaStream_t)stream>>>(s_obs, s_act, s_rew, s_next, s_term, obs, act, rew, next_obs, term, n, od, ad, cap, state);
  rpm_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, n, cap);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_rpm_sample_cursor(const float* s_obs, const float* s_act, const float* s_rew, const float* s_next, const float* s_term, float* obs, float* act, float* rew,
                          float* next_obs, float* term, int batch, int od, int ad, uint64_t seed, long long* state, void* stream) {
  if (!s_obs || !obs || !state || batch < 1) return -1;
  rpm_sample_cursor_kernel<<<batch, 64, 0, (cudaStream_t)stream>>>(s_obs, s_act, s_rew, s_next, s_term, obs, act, rew, next_obs, term, batch, od, ad, seed, state);
  rpm_count_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_rpm_append_masked_cursor(float* s_obs, float* s_act, float* s_rew, float* s_next, float* s_term, const float* obs, const float* act, const float* rew,
                                 const float* next_obs, const float* term, const uint8_t* valid, int n, int od, int ad, int cap, long long* state, void* stream) {
  if (!s_obs || !s_act || !s_rew || !s_next || !s_term || !obs || !act || !rew || !next_obs || !term || !valid || !state || n < 1 || cap < n) return -1;
  const int tile = 32 * ((n + 32 * MASK_MAX_CTAS - 1) / (32 * MASK_MAX_CTAS));
  rpm_append_masked_kernel<<<(n + tile - 1) / tile, MASK_THREADS, 0, (cudaStream_t)stream>>>(s_obs, s_act, s_rew, s_next, s_term, obs, act, rew, next_obs, term,
                                                                                            valid, n, od, ad, cap, tile, state);
  rpm_advance_masked_kernel<<<1, MASK_THREADS, 0, (cudaStream_t)stream>>>(state, valid, n, cap);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_bc_observe(const float* obs, int n, int obs_dim, float* student, float* ring_obs, float* ring_ref, int pos, int cap, uint32_t seed, uint32_t step,
                   int noise, void* stream) {
  if (!obs || !student || n < 1 || obs_dim < 37 || (!ring_obs) != (!ring_ref)) return -1;
  if (ring_ref && (cap < n || pos < 0)) return -1;
  const size_t total = (size_t)n * obs_dim;
  const int grid = (int)std::min<size_t>((total + BC_THREADS - 1) / BC_THREADS, 8192);
  bc_observe_kernel<<<grid, BC_THREADS, 0, (cudaStream_t)stream>>>(obs, n, obs_dim, student, ring_obs, ring_ref, pos, cap,
                                                                   (uint64_t)seed | ((uint64_t)step << 32), noise);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
int b2q_bc_gather_cursor(const float* ring_obs, const float* ring_ref, const int64_t* perm, int perm_len, long long* state, float* out_obs, float* out_ref,
                         int batch, int obs_dim, int ref_dim, void* stream) {
  if (!ring_obs || !ring_ref || !perm || !state || !out_obs || !out_ref || batch < 1 || obs_dim < 1 || ref_dim < 1 || perm_len < 0) return -1;
  const int grid = std::min((batch * (obs_dim + ref_dim) + BC_THREADS - 1) / BC_THREADS, 4096);
  bc_gather_kernel<<<grid, BC_THREADS, 0, (cudaStream_t)stream>>>(ring_obs, ring_ref, perm, perm_len, state, out_obs, out_ref, batch, obs_dim, ref_dim);
  bc_cursor_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, batch);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
}
