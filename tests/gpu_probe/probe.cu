// probe.cu — device probe of the step kernel's float32 primitives.  TEST INFRASTRUCTURE ONLY (built by tests/gpu_probe/probe.py into
// tests/gpu_probe/_build/libb2q_probe.so, never loaded by the product package).
//
// Exhaustive sweeps: every thread makes its float input from its own index, evaluates the product function (b2q_math.cuh, device branch)
// and a float64 reference on the device, and each block reduces its worst error and its arg-max, so a few numbers per block come back.
// Map kernels: one thread per element of a host-given input array (prim.h), for the sampled and edge-case checks.
// Philox: b2q::philox4 and b2q_philox::philox_normal against the CUDA toolkit's curand_Philox4x32_10.
//
// The C entry points take host pointers, copy through device buffers they own and return a cudaError_t code.  Every kernel bounds-checks
// its index and touches only its own buffers.
#include <cfloat>
#include <cstdint>
#include <cuda_runtime.h>
#include <curand_philox4x32_x.h>
#include "prim.h"
#include "../../paddlerobotics_b200/csrc/b2q_philox.cuh"

using namespace b2q;
using namespace b2q_prim;

namespace {

constexpr int TPB = 256;

// |got - ref| in units of the float32 ulp of ref (floored at the smallest normal's ulp, 2^-149); a non-NaN ref with a NaN or infinite
// got counts as infinitely wrong, a NaN ref with a NaN got as exact
__device__ double ulp_err(float got, double ref) {
  if (ref != ref) return got != got ? 0.0 : INFINITY;
  if (got != got || (isinf(got) && !isinf(ref))) return INFINITY;
  if (isinf(ref)) return (double)got == ref ? 0.0 : INFINITY;
  int e; frexp(fmax(fabs(ref), (double)FLT_MIN), &e);
  return fabs((double)got - ref) / ldexp(1.0, e - 24);
}

struct SincosOp {   // err0 = sin, err1 = cos, flag: s^2 + c^2 off 1 by more than 4 ulp
  __device__ void operator()(float x, double& e0, double& e1, int& flag) const {
    float s, c; sincos_f(x, &s, &c);
    e0 = ulp_err(s, sin((double)x)); e1 = ulp_err(c, cos((double)x));
    flag = fabs((double)s * s + (double)c * c - 1.0) > 4.0 * FLT_EPSILON;
  }
};
struct RcpOp {      // err0 = ulp error where x and 1/x are normal; err1 = 1 where an edge input misses its documented value; flag = not the correctly rounded 1/x
  __device__ void operator()(float x, double& e0, double& e1, int& flag) const {
    float r = rcp_f(x); double ax = fabs((double)x);
    e0 = e1 = 0; flag = 0;
    if (ax >= (double)FLT_MIN && ax <= 0x1p126) { e0 = ulp_err(r, 1.0 / (double)x); flag = r != __frcp_rn(x); }
    else if (ax < (double)FLT_MIN) e1 = (r == r);                                      // subnormal: NaN (rcp.approx.ftz gives inf, the Newton step inf - inf)
    else e1 = !(r == 0.0f && signbit(r) == signbit(x));                               // |x| > 2^126: signed zero (the approximation flushes to zero)
  }
};
struct RsqrtOp {    // err0 = ulp error against 1/sqrt(x); flag = differs from the host branch 1.0f / sqrtf(x)
  __device__ void operator()(float x, double& e0, double& e1, int& flag) const {
    float r = rsqrt_f(x);
    e0 = ulp_err(r, 1.0 / sqrt((double)x)); e1 = 0;
    flag = r != __fdiv_rn(1.0f, __fsqrt_rn(x));
  }
};

// inputs: bit patterns lo..hi (inclusive), and the same with the sign bit set when `both`
template <class Op>
__global__ void __launch_bounds__(TPB) k_sweep(uint32_t lo, uint32_t hi, int both, Op op, double* err, uint32_t* arg, unsigned long long* cnt, int nblk) {
  __shared__ double se[2][TPB];
  __shared__ uint32_t sa[2][TPB];
  __shared__ unsigned long long sc[TPB];
  const uint64_t per = (uint64_t)(hi - lo) + 1, total = both ? 2 * per : per;
  double e0 = -1, e1 = -1; uint32_t a0 = 0, a1 = 0; unsigned long long c = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * TPB + threadIdx.x; i < total; i += (uint64_t)gridDim.x * TPB) {
    uint32_t bits = i < per ? lo + (uint32_t)i : (lo + (uint32_t)(i - per)) | 0x80000000u;
    double r0, r1; int f;
    op(__uint_as_float(bits), r0, r1, f);
    if (r0 > e0) { e0 = r0; a0 = bits; }
    if (r1 > e1) { e1 = r1; a1 = bits; }
    c += f;
  }
  const int t = threadIdx.x;
  se[0][t] = e0; se[1][t] = e1; sa[0][t] = a0; sa[1][t] = a1; sc[t] = c;
  __syncthreads();
  for (int s = TPB / 2; s > 0; s >>= 1) {
    if (t < s) {
      for (int k = 0; k < 2; k++) if (se[k][t + s] > se[k][t]) { se[k][t] = se[k][t + s]; sa[k][t] = sa[k][t + s]; }
      sc[t] += sc[t + s];
    }
    __syncthreads();
  }
  if (t == 0 && (int)blockIdx.x < nblk) {
    err[2 * blockIdx.x] = se[0][0]; err[2 * blockIdx.x + 1] = se[1][0];
    arg[2 * blockIdx.x] = sa[0][0]; arg[2 * blockIdx.x + 1] = sa[1][0]; cnt[blockIdx.x] = sc[0];
  }
}

// ---- Philox: tuple i -> (key, counter); a quarter of the keys have only a low word, an eighth of the counters are all 0 or all ones
__device__ uint32_t mix32(uint32_t x) { x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16; return x; }
__device__ void tuple_of(uint32_t i, uint64_t& seed, uint32_t& c0, uint32_t& c1, uint32_t& c2) {
  uint32_t k0 = mix32(i ^ 0x1234567u), k1 = mix32(i * 3u + 0x89ABCDEu);
  if ((i & 3) == 0) k1 = 0;
  seed = ((uint64_t)k1 << 32) | k0;
  c0 = i; c1 = mix32(i + 0x9E3779B9u); c2 = mix32(~i);
  if ((i & 7) == 1) c0 = c1 = c2 = 0;
  if ((i & 7) == 5) c0 = c1 = c2 = 0xFFFFFFFFu;
}
// Box-Muller of four words in float64: u = (r >> 8) + 0.5, scaled by 2^-24, either exactly (uexact) or as the float32 path rounds it
__device__ void bm64(const uint32_t r[4], bool uexact, double n[4], double rad[2]) {
  double u[4];
  for (int k = 0; k < 4; k++) u[k] = uexact ? ((double)(r[k] >> 8) + 0.5) * 0x1p-24 : (double)(((float)(r[k] >> 8) + 0.5f) * 0x1p-24f);
  const double tp = 6.283185307179586476925286766559;
  rad[0] = sqrt(-2 * log(u[0])); rad[1] = sqrt(-2 * log(u[2]));
  n[0] = rad[0] * cos(tp * u[1]); n[1] = rad[0] * sin(tp * u[1]); n[2] = rad[1] * cos(tp * u[3]); n[3] = rad[1] * sin(tp * u[3]);
}
// per block, PH_N values: [0] philox4 words != curand, [1] philox_normal != the float32 formula on curand's words (counter (row, col,
// 0x9E3779B9, 0)), [2] normal4<float> rel. error vs float64 of its own float32-rounded u, in eps32 x max(1, radius), [3] normal4<float>
// abs. error vs exact u, [4] normal4<double> rel. error in eps64 x max(1, radius), [5] philox_normal rel. error (as [2]), [6] philox_normal
// abs. error vs exact u, [7] first tuple index with a word mismatch (or 2^32)
constexpr int PH_N = 8;
__global__ void __launch_bounds__(TPB) k_philox(uint32_t n, double* out, int nblk) {
  __shared__ double sm[PH_N][TPB];
  double v[PH_N] = {0, 0, 0, 0, 0, 0, 0, 4294967296.0};
  for (uint64_t ii = (uint64_t)blockIdx.x * TPB + threadIdx.x; ii < n; ii += (uint64_t)gridDim.x * TPB) {
    const uint32_t i = (uint32_t)ii;
    uint64_t seed; uint32_t c0, c1, c2; tuple_of(i, seed, c0, c1, c2);
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    uint32_t w[4]; philox4(seed, c0, c1, c2, w);
    const uint4 ref = curand_Philox4x32_10(make_uint4(c0, c1, c2, 0u), key);
    const uint32_t rr[4] = {ref.x, ref.y, ref.z, ref.w};
    const bool bad = w[0] != ref.x || w[1] != ref.y || w[2] != ref.z || w[3] != ref.w;
    v[0] += bad;
    if (bad && (double)i < v[7]) v[7] = i;
    // b2q_philox: counter (row, col, 0x9E3779B9, 0), words 0 and 1 through its own float32 Box-Muller
    const uint4 rm = curand_Philox4x32_10(make_uint4(c0, c1, 0x9E3779B9u, 0u), key);
    const float pn = b2q_philox::philox_normal(seed, c0, c1);
    const float pu1 = ((float)(rm.x >> 8) + 0.5f) * (1.0f / 16777216.0f), pu2 = ((float)(rm.y >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float pf = sqrtf(-2.0f * logf(pu1)) * cosf(6.283185307179586f * pu2);
    v[1] += __float_as_uint(pn) != __float_as_uint(pf);
    {
      const uint32_t rm4[4] = {rm.x, rm.y, 0u, 0u};
      double nr[4], rad[2], ne[4], rade[2];
      bm64(rm4, false, nr, rad); bm64(rm4, true, ne, rade);
      v[5] = fmax(v[5], fabs((double)pn - nr[0]) / (FLT_EPSILON * fmax(1.0, rad[0])));
      v[6] = fmax(v[6], fabs((double)pn - ne[0]));
    }
    float nf[4]; philox_normal4<float>(seed, c0, c1, c2, nf);
    double nd[4]; philox_normal4<double>(seed, c0, c1, c2, nd);
    double nr[4], rad[2], ne[4], rade[2];
    bm64(rr, false, nr, rad); bm64(rr, true, ne, rade);
    for (int k = 0; k < 4; k++) {
      v[2] = fmax(v[2], fabs((double)nf[k] - nr[k]) / (FLT_EPSILON * fmax(1.0, rad[k / 2])));
      v[3] = fmax(v[3], fabs((double)nf[k] - ne[k]));
      v[4] = fmax(v[4], fabs(nd[k] - ne[k]) / (DBL_EPSILON * fmax(1.0, rade[k / 2])));
    }
  }
  const int t = threadIdx.x;
  for (int k = 0; k < PH_N; k++) sm[k][t] = v[k];
  __syncthreads();
  for (int s = TPB / 2; s > 0; s >>= 1) {
    if (t < s) {
      sm[0][t] += sm[0][t + s]; sm[1][t] += sm[1][t + s];
      for (int k = 2; k < 7; k++) sm[k][t] = fmax(sm[k][t], sm[k][t + s]);
      sm[7][t] = fmin(sm[7][t], sm[7][t + s]);
    }
    __syncthreads();
  }
  if (t == 0 && (int)blockIdx.x < nblk) for (int k = 0; k < PH_N; k++) out[(size_t)blockIdx.x * PH_N + k] = sm[k][0];
}

// ---- map kernels: one thread per element
__global__ void k_sincos_map(int n, const float* a, float* s, float* c, double* ds, double* dc) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  sincos_f(a[i], s + i, c + i);
  ds[i] = sin((double)a[i]); dc[i] = cos((double)a[i]);
}
__global__ void k_unary_map(int n, int which, const float* x, float* y) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  y[i] = which == 0 ? rcp_f(x[i]) : rsqrt_f(x[i]);
}
template <typename T> __global__ void k_leg_map(int n, int inverse, const Model<T>* md, const int* leg, const T* in, T* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int k = leg[i];
  if (k < 0 || k > 3) return;
  if (inverse) leg_inv(*md, k, in + 3 * (size_t)i, out + 3 * (size_t)i); else leg_fk(*md, k, in + 3 * (size_t)i, out + 3 * (size_t)i);
}
template <typename T> __global__ void k_rpy_map(int n, const T* q, T* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rpy(q + 4 * (size_t)i, out + 3 * (size_t)i);
}
template <typename T> __global__ void k_terrain_map(int n, Cfg<T> cf, const T* xy, T* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) terrain(cf, xy[2 * (size_t)i], xy[2 * (size_t)i + 1], out + 4 * (size_t)i);
}
template <typename T> __global__ void k_solve_map(int n, const T* S, const T* b, T* x) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) spd_solve(S + 21 * (size_t)i, b + 6 * (size_t)i, x + 6 * (size_t)i);
}

// ---- host side: device buffers owned by one call
struct Bufs {
  void* p[8]; int k = 0; cudaError_t err = cudaSuccess;
  template <typename T> T* alloc(size_t n) { void* d = nullptr; if (err == cudaSuccess) err = cudaMalloc(&d, n * sizeof(T) + 16); p[k++] = d; return (T*)d; }
  template <typename T> T* up(const T* h, size_t n) { T* d = alloc<T>(n); if (err == cudaSuccess) err = cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice); return d; }
  template <typename T> void down(T* h, const T* d, size_t n) { if (err == cudaSuccess) err = cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost); }
  int done() {
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    return (int)err;
  }
  ~Bufs() { for (int i = 0; i < k; i++) if (p[i]) cudaFree(p[i]); }
};
inline int grid(int n) { return (n + TPB - 1) / TPB; }

template <class Op>
int sweep(Op op, uint32_t lo, uint32_t hi, int both, int nblk, double* err, uint32_t* arg, unsigned long long* cnt) {
  if (nblk < 1 || hi < lo) return (int)cudaErrorInvalidValue;
  Bufs b;
  double* de = b.alloc<double>(2 * (size_t)nblk); uint32_t* da = b.alloc<uint32_t>(2 * (size_t)nblk); unsigned long long* dc = b.alloc<unsigned long long>(nblk);
  if (b.err == cudaSuccess) k_sweep<<<nblk, TPB>>>(lo, hi, both, op, de, da, dc, nblk);
  if (b.err == cudaSuccess) b.err = cudaGetLastError();
  b.down(err, de, 2 * (size_t)nblk); b.down(arg, da, 2 * (size_t)nblk); b.down(cnt, dc, nblk);
  return b.done();
}
template <typename T>
int leg_map(int n, int inverse, const int* leg, const T* in, T* out) {
  Bufs b;
  Model<T> md = default_model<T>();
  Model<T>* dm = b.up(&md, 1);
  int* dl = b.up(leg, n); T* di = b.up(in, 3 * (size_t)n); T* dout = b.alloc<T>(3 * (size_t)n);
  if (b.err == cudaSuccess) k_leg_map<T><<<grid(n), TPB>>>(n, inverse, dm, dl, di, dout);
  b.down(out, dout, 3 * (size_t)n);
  return b.done();
}
template <typename T>
int rpy_map(int n, const T* q, T* out) {
  Bufs b;
  T* dq = b.up(q, 4 * (size_t)n); T* dout = b.alloc<T>(3 * (size_t)n);
  if (b.err == cudaSuccess) k_rpy_map<T><<<grid(n), TPB>>>(n, dq, dout);
  b.down(out, dout, 3 * (size_t)n);
  return b.done();
}
template <typename T>
int terrain_map(int nx, int ny, double x0, double y0, double cell, const double* hf, int n, const T* xy, T* out) {
  if (nx < 2 || ny < 2 || !(cell > 0)) return (int)cudaErrorInvalidValue;
  Bufs b;
  T* h = new T[(size_t)nx * ny];
  for (size_t i = 0; i < (size_t)nx * ny; i++) h[i] = (T)hf[i];
  T* dh = b.up(h, (size_t)nx * ny);
  delete[] h;
  T* dxy = b.up(xy, 2 * (size_t)n); T* dout = b.alloc<T>(4 * (size_t)n);
  if (b.err == cudaSuccess) k_terrain_map<T><<<grid(n), TPB>>>(n, hf_cfg<T>(nx, ny, x0, y0, cell, dh), dxy, dout);
  b.down(out, dout, 4 * (size_t)n);
  return b.done();
}
template <typename T>
int solve_map(int n, const T* S, const T* rhs, T* x) {
  Bufs b;
  T* dS = b.up(S, 21 * (size_t)n); T* db = b.up(rhs, 6 * (size_t)n); T* dx = b.alloc<T>(6 * (size_t)n);
  if (b.err == cudaSuccess) k_solve_map<T><<<grid(n), TPB>>>(n, dS, db, dx);
  b.down(x, dx, 6 * (size_t)n);
  return b.done();
}

}  // namespace

extern "C" {
// which: 0 = m_sincos, 1 = m_rcp, 2 = m_rsqrt; err/arg: [nblk][2], cnt: [nblk]
int probe_sweep(int which, uint32_t lo, uint32_t hi, int both, int nblk, double* err, uint32_t* arg, unsigned long long* cnt) {
  if (which == 0) return sweep(SincosOp{}, lo, hi, both, nblk, err, arg, cnt);
  if (which == 1) return sweep(RcpOp{}, lo, hi, both, nblk, err, arg, cnt);
  if (which == 2) return sweep(RsqrtOp{}, lo, hi, both, nblk, err, arg, cnt);
  return (int)cudaErrorInvalidValue;
}
// out: [nblk][8], see k_philox
int probe_philox(uint32_t n, int nblk, double* out) {
  if (nblk < 1) return (int)cudaErrorInvalidValue;
  Bufs b;
  double* d = b.alloc<double>((size_t)nblk * PH_N);
  if (b.err == cudaSuccess) k_philox<<<nblk, TPB>>>(n, d, nblk);
  if (b.err == cudaSuccess) b.err = cudaGetLastError();
  b.down(out, d, (size_t)nblk * PH_N);
  return b.done();
}
int probe_sincos(int n, const float* a, float* s, float* c, double* ds, double* dc) {
  Bufs b;
  float* da = b.up(a, n); float* d_s = b.alloc<float>(n); float* d_c = b.alloc<float>(n); double* d_ds = b.alloc<double>(n); double* d_dc = b.alloc<double>(n);
  if (b.err == cudaSuccess) k_sincos_map<<<grid(n), TPB>>>(n, da, d_s, d_c, d_ds, d_dc);
  b.down(s, d_s, n); b.down(c, d_c, n); b.down(ds, d_ds, n); b.down(dc, d_dc, n);
  return b.done();
}
int probe_unary(int which, int n, const float* x, float* y) {
  Bufs b;
  float* dx = b.up(x, n); float* dy = b.alloc<float>(n);
  if (b.err == cudaSuccess) k_unary_map<<<grid(n), TPB>>>(n, which, dx, dy);
  b.down(y, dy, n);
  return b.done();
}
int probe_leg(int prec, int n, int inverse, const int* leg, const void* in, void* out) {
  return prec ? leg_map<double>(n, inverse, leg, (const double*)in, (double*)out) : leg_map<float>(n, inverse, leg, (const float*)in, (float*)out);
}
int probe_rpy(int prec, int n, const void* q, void* out) {
  return prec ? rpy_map<double>(n, (const double*)q, (double*)out) : rpy_map<float>(n, (const float*)q, (float*)out);
}
int probe_terrain(int prec, int nx, int ny, double x0, double y0, double cell, const double* hf, int n, const void* xy, void* out) {
  return prec ? terrain_map<double>(nx, ny, x0, y0, cell, hf, n, (const double*)xy, (double*)out)
              : terrain_map<float>(nx, ny, x0, y0, cell, hf, n, (const float*)xy, (float*)out);
}
int probe_solve(int prec, int n, const void* S, const void* rhs, void* x) {
  return prec ? solve_map<double>(n, (const double*)S, (const double*)rhs, (double*)x) : solve_map<float>(n, (const float*)S, (const float*)rhs, (float*)x);
}
}
