// b2q_math.cuh — small fixed-size algebra used by the A1 step kernels (sm_90a) and by the host SIMT
// emulation harness in tests/emu (same source, different Comm policy).
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define B2Q_HD __host__ __device__ __forceinline__
#define B2Q_D __device__ __forceinline__
#else
#define B2Q_HD inline
#define B2Q_D inline
#endif

namespace b2q {

// ---- scalar math wrappers (precise variants: no fast-math intrinsics, parity with the f64 oracle matters)
B2Q_HD float m_sqrt(float x) { return sqrtf(x); }
B2Q_HD double m_sqrt(double x) { return sqrt(x); }
// m_rsqrt(float): rsqrtf on the device, <= 1.52 ulp over every positive normal float (measured exhaustively on H100, tests/gpu_probe); the
// host build's 1.0f / sqrtf(x) rounds twice, <= 1.48 ulp, and differs from the device in about a third of the inputs.  Callers: chol6's
// pivots, terrain normals, contact tangents and the quaternion renormalisation, all positive and normal.
#if defined(__CUDA_ARCH__)
B2Q_HD float m_rsqrt(float x) { return rsqrtf(x); }
#else
B2Q_HD float m_rsqrt(float x) { return 1.0f / sqrtf(x); }
#endif
B2Q_HD double m_rsqrt(double x) { return 1.0 / sqrt(x); }
B2Q_HD float m_sin(float x) { return sinf(x); }
B2Q_HD double m_sin(double x) { return sin(x); }
B2Q_HD float m_cos(float x) { return cosf(x); }
B2Q_HD double m_cos(double x) { return cos(x); }
B2Q_HD float m_acos(float x) { return acosf(x); }
B2Q_HD double m_acos(double x) { return acos(x); }
B2Q_HD float m_asin(float x) { return asinf(x); }
B2Q_HD double m_asin(double x) { return asin(x); }
B2Q_HD float m_atan2(float y, float x) { return atan2f(y, x); }
B2Q_HD double m_atan2(double y, double x) { return atan2(y, x); }
B2Q_HD float m_exp(float x) { return expf(x); }
B2Q_HD double m_exp(double x) { return exp(x); }
B2Q_HD float m_tanh(float x) { return tanhf(x); }
B2Q_HD double m_tanh(double x) { return tanh(x); }
B2Q_HD float m_fmod(float x, float y) { return fmodf(x, y); }
B2Q_HD double m_fmod(double x, double y) { return fmod(x, y); }
B2Q_HD float m_abs(float x) { return fabsf(x); }
B2Q_HD double m_abs(double x) { return fabs(x); }
B2Q_HD float m_min(float a, float b) { return fminf(a, b); }
B2Q_HD double m_min(double a, double b) { return fmin(a, b); }
B2Q_HD float m_max(float a, float b) { return fmaxf(a, b); }
B2Q_HD double m_max(double a, double b) { return fmax(a, b); }
B2Q_HD float m_fma(float a, float b, float c) { return fmaf(a, b, c); }
B2Q_HD double m_fma(double a, double b, double c) { return fma(a, b, c); }
B2Q_HD bool m_isfinite(float x) { return (x - x) == 0.0f; }
B2Q_HD bool m_isfinite(double x) { return (x - x) == 0.0; }
B2Q_HD bool m_isnan(float x) { return x != x; }
B2Q_HD bool m_isnan(double x) { return x != x; }

B2Q_HD float m_log(float x) { return logf(x); }
B2Q_HD double m_log(double x) { return log(x); }

// counter-based Gaussian for sensor noise: Philox4x32-10 keyed by the 64-bit seed, counter (c0,c1,c2,0) -> 4 x u32 -> two Box-Muller
// pairs.  Integer part identical on host and device; the transform is evaluated in T.
B2Q_HD uint32_t mulhi32(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32); }
B2Q_HD void philox4(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t out[4]) {
  uint32_t c3 = 0, k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  for (int i = 0; i < 10; i++) {
    uint32_t h0 = mulhi32(0xD2511F53u, c0), l0 = 0xD2511F53u * c0, h1 = mulhi32(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    uint32_t n0 = h1 ^ c1 ^ k0, n2 = h0 ^ c3 ^ k1;
    c0 = n0; c1 = l1; c2 = n2; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
template <typename T> B2Q_HD void philox_normal4(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, T n[4]) {
  uint32_t r[4]; philox4(seed, c0, c1, c2, r);
  const T two_pi = T(6.283185307179586476925286766559), sc = T(1.0 / 16777216.0);
  T u0 = (T(r[0] >> 8) + T(0.5)) * sc, u1 = (T(r[1] >> 8) + T(0.5)) * sc, u2 = (T(r[2] >> 8) + T(0.5)) * sc, u3 = (T(r[3] >> 8) + T(0.5)) * sc;
  T ra = m_sqrt(T(-2) * m_log(u0)), rb = m_sqrt(T(-2) * m_log(u2));
  n[0] = ra * m_cos(two_pi * u1); n[1] = ra * m_sin(two_pi * u1); n[2] = rb * m_cos(two_pi * u3); n[3] = rb * m_sin(two_pi * u3);
}

// reciprocal: one MUFU.RCP + one Newton step on the GPU (no slow path / branch); exact division elsewhere.  Measured exhaustively on H100
// (tests/gpu_probe): for every normal x with |x| <= 2^126 the device result is the correctly rounded 1/x, the host's.  The edges follow
// from rcp.approx.ftz: x = +-0, +-inf and subnormal x give NaN (the Newton step computes 0 * inf or inf - inf), |x| > 2^126 gives a
// signed zero instead of the subnormal 1/x.  No caller uses them: det of the 3x3 joint-space block and W_ii of an active contact
// row are positive and far inside the normal range, and 1/th is used only for th >= 1e-4 (the substep computes 1/W_ii of inactive rows and
// 1/th for every th, and selects them away).
#if defined(__CUDA_ARCH__)
B2Q_HD float m_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return fmaf(r, fmaf(-x, r, 1.0f), r); }
#else
B2Q_HD float m_rcp(float x) { return 1.0f / x; }
#endif
B2Q_HD double m_rcp(double x) { return 1.0 / x; }

// sin and cos together for |a| up to a few turns (joint angles, Euler-step rotation angles): Cody-Waite reduction by
// pi/2 (3 constants) + the classic degree-7/8 minimax kernels on [-pi/4, pi/4]; branch-free, ~30 instructions
// (libm's sinf/cosf carry a Payne-Hanek slow path that costs >2000 instructions of code in this kernel).
// Measured over all 2.2e9 floats in [-8 pi, 8 pi] on H100 (tests/gpu_probe): <= 1.50 ulp for sin, <= 1.49 ulp for cos, the host
// build bit-identical.  Sampled up to |a| = 2^20 the outputs stay finite with s^2 + c^2 within 1.5 eps of 1; NaN and +-inf give NaN.
// The callers need |a| < 8 pi: leg_kin's q1, q2 and q1 + q2 (|q1 + q2| < 6.9 over the URDF ranges) and the Euler step's |w| dt / 2.
B2Q_HD void m_sincos(float a, float& s, float& c) {
  float q = rintf(a * 0.636619772367581343f);            // nearest multiple of pi/2
  int n = (int)q;
  float r = fmaf(q, -1.57079601287841796875f, a);        // pi/2 split in three parts
  r = fmaf(q, -3.1391647326017846353352069854736328125e-7f, r);
  r = fmaf(q, -5.390302529957764765543e-15f, r);
  float r2 = r * r;
  float sp = fmaf(fmaf(fmaf(-1.95152959e-4f, r2, 8.33216087e-3f), r2, -1.66666546e-1f), r2 * r, r);
  float cp = fmaf(fmaf(fmaf(fmaf(2.44331571e-5f, r2, -1.38873163e-3f), r2, 4.16666457e-2f), r2, -0.5f), r2, 1.0f);
  float ss = (n & 1) ? cp : sp, cc = (n & 1) ? sp : cp;
  s = (n & 2) ? -ss : ss;
  c = ((n + 1) & 2) ? -cc : cc;
}
B2Q_HD void m_sincos(double a, double& s, double& c) { s = sin(a); c = cos(a); }

template <typename T>
struct V3 {
  T x, y, z;
};
template <typename T> B2Q_HD V3<T> mk(T x, T y, T z) { V3<T> r; r.x = x; r.y = y; r.z = z; return r; }
template <typename T> B2Q_HD V3<T> operator+(V3<T> a, V3<T> b) { return mk<T>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename T> B2Q_HD V3<T> operator-(V3<T> a, V3<T> b) { return mk<T>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename T> B2Q_HD V3<T> operator-(V3<T> a) { return mk<T>(-a.x, -a.y, -a.z); }
template <typename T> B2Q_HD V3<T> operator*(V3<T> a, T s) { return mk<T>(a.x * s, a.y * s, a.z * s); }
template <typename T> B2Q_HD V3<T> operator*(T s, V3<T> a) { return mk<T>(a.x * s, a.y * s, a.z * s); }
template <typename T> B2Q_HD T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> B2Q_HD V3<T> cross(V3<T> a, V3<T> b) { return mk<T>(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// symmetric 3x3
template <typename T>
struct S3 {
  T xx, xy, xz, yy, yz, zz;
};
template <typename T> B2Q_HD V3<T> mul(const S3<T>& s, V3<T> v) {
  return mk<T>(s.xx * v.x + s.xy * v.y + s.xz * v.z, s.xy * v.x + s.yy * v.y + s.yz * v.z, s.xz * v.x + s.yz * v.y + s.zz * v.z);
}
template <typename T> B2Q_HD S3<T> operator+(const S3<T>& a, const S3<T>& b) { S3<T> r = {a.xx + b.xx, a.xy + b.xy, a.xz + b.xz, a.yy + b.yy, a.yz + b.yz, a.zz + b.zz}; return r; }
// m (|c|^2 1 - c c^T)
template <typename T> B2Q_HD S3<T> point_inertia(T m, V3<T> c) {
  S3<T> r = {m * (c.y * c.y + c.z * c.z), -m * c.x * c.y, -m * c.x * c.z, m * (c.x * c.x + c.z * c.z), -m * c.y * c.z, m * (c.x * c.x + c.y * c.y)};
  return r;
}

// rotation matrix stored by columns (body->outer): v_outer = cx*v.x + cy*v.y + cz*v.z
template <typename T>
struct R3 {
  V3<T> cx, cy, cz;
};
template <typename T> B2Q_HD V3<T> rot(const R3<T>& R, V3<T> v) { return R.cx * v.x + R.cy * v.y + R.cz * v.z; }
template <typename T> B2Q_HD V3<T> rotT(const R3<T>& R, V3<T> v) { return mk<T>(dot(R.cx, v), dot(R.cy, v), dot(R.cz, v)); }
template <typename T> B2Q_HD S3<T> rot_sym(const R3<T>& R, const S3<T>& I) {  // R I R^T
  V3<T> a = R.cx * I.xx + R.cy * I.xy + R.cz * I.xz;  // (R I) column 0
  V3<T> b = R.cx * I.xy + R.cy * I.yy + R.cz * I.yz;
  V3<T> c = R.cx * I.xz + R.cy * I.yz + R.cz * I.zz;
  // out = [a b c] R^T = a cx^T + b cy^T + c cz^T
  S3<T> o;
  o.xx = a.x * R.cx.x + b.x * R.cy.x + c.x * R.cz.x;
  o.xy = a.x * R.cx.y + b.x * R.cy.y + c.x * R.cz.y;
  o.xz = a.x * R.cx.z + b.x * R.cy.z + c.x * R.cz.z;
  o.yy = a.y * R.cx.y + b.y * R.cy.y + c.y * R.cz.y;
  o.yz = a.y * R.cx.z + b.y * R.cy.z + c.y * R.cz.z;
  o.zz = a.z * R.cx.z + b.z * R.cy.z + c.z * R.cz.z;
  return o;
}
template <typename T> B2Q_HD R3<T> quat_to_R(T x, T y, T z, T w) {  // xyzw, body->world (pybullet convention)
  R3<T> R;
  R.cx = mk<T>(1 - 2 * (y * y + z * z), 2 * (x * y + z * w), 2 * (x * z - y * w));
  R.cy = mk<T>(2 * (x * y - z * w), 1 - 2 * (x * x + z * z), 2 * (y * z + x * w));
  R.cz = mk<T>(2 * (x * z + y * w), 2 * (y * z - x * w), 1 - 2 * (x * x + y * y));
  return R;
}
template <typename T> B2Q_HD V3<T> quat_to_rpy(T x, T y, T z, T w) {  // minitaur.py:613-621 (getEulerFromQuaternion)
  T s = 2 * (w * y - z * x);
  s = m_min(m_max(s, T(-1)), T(1));
  return mk<T>(m_atan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y)), m_asin(s), m_atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z)));
}

// 6-vectors [ang; lin]
template <typename T>
struct V6 {
  V3<T> a, l;
};
template <typename T> B2Q_HD V6<T> operator+(V6<T> p, V6<T> q) { V6<T> r; r.a = p.a + q.a; r.l = p.l + q.l; return r; }
template <typename T> B2Q_HD V6<T> operator-(V6<T> p, V6<T> q) { V6<T> r; r.a = p.a - q.a; r.l = p.l - q.l; return r; }
template <typename T> B2Q_HD V6<T> operator*(V6<T> p, T s) { V6<T> r; r.a = p.a * s; r.l = p.l * s; return r; }
template <typename T> B2Q_HD T dot6(V6<T> p, V6<T> q) { return dot(p.a, q.a) + dot(p.l, q.l); }
template <typename T> B2Q_HD T get6(const V6<T>& v, int i) { return i == 0 ? v.a.x : i == 1 ? v.a.y : i == 2 ? v.a.z : i == 3 ? v.l.x : i == 4 ? v.l.y : v.l.z; }

// packed lower-triangular 6x6 / symmetric 6x6: index (i>=j) -> i*(i+1)/2 + j
B2Q_HD constexpr int tri(int i, int j) { return i >= j ? i * (i + 1) / 2 + j : j * (j + 1) / 2 + i; }

// Cholesky of a packed symmetric 6x6 (lower).  Out: L (lower, unit scaling NOT applied) and the reciprocals of its
// diagonal in Li[6], so that the triangular solves below are multiply-only (no division on their serial chains).
template <typename T> B2Q_HD void chol6(T* S /*21, in: sym lower; out: L lower*/, T* Li /*6*/) {
#pragma unroll
  for (int j = 0; j < 6; j++) {
    T d = S[tri(j, j)];
#pragma unroll
    for (int k = 0; k < j; k++) d -= S[tri(j, k)] * S[tri(j, k)];
    T inv = m_rsqrt(d);
    S[tri(j, j)] = d * inv;
    Li[j] = inv;
#pragma unroll
    for (int i = j + 1; i < 6; i++) {
      T s = S[tri(i, j)];
#pragma unroll
      for (int k = 0; k < j; k++) s -= S[tri(i, k)] * S[tri(j, k)];
      S[tri(i, j)] = s * inv;
    }
  }
}
template <typename T> B2Q_HD void fwd6(const T* L, const T* Li, T* b) {  // b <- L^-1 b
#pragma unroll
  for (int i = 0; i < 6; i++) {
    T s = b[i];
#pragma unroll
    for (int k = 0; k < i; k++) s -= L[tri(i, k)] * b[k];
    b[i] = s * Li[i];
  }
}
template <typename T> B2Q_HD void bwd6(const T* L, const T* Li, T* b) {  // b <- L^-T b
#pragma unroll
  for (int i = 5; i >= 0; i--) {
    T s = b[i];
#pragma unroll
    for (int k = i + 1; k < 6; k++) s -= L[tri(k, i)] * b[k];
    b[i] = s * Li[i];
  }
}
template <typename T> B2Q_HD void v6_to_arr(const V6<T>& v, T* a) { a[0] = v.a.x; a[1] = v.a.y; a[2] = v.a.z; a[3] = v.l.x; a[4] = v.l.y; a[5] = v.l.z; }
template <typename T> B2Q_HD V6<T> arr_to_v6(const T* a) { V6<T> v; v.a = mk<T>(a[0], a[1], a[2]); v.l = mk<T>(a[3], a[4], a[5]); return v; }

}  // namespace b2q
