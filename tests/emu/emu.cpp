// emu.cpp — CPU SIMT-emulation harness of the DEVICE code in paddlerobotics_b200/csrc/b2q_sim.cuh.
//
// TEST INFRASTRUCTURE ONLY (built by tests/emu/Makefile into tests/emu/_build/libb2q_emu.so, never shipped, never
// loaded by the product package).  It compiles the very same templated lane functions the CUDA kernels call, with
// the `Comm` policy replaced by a 4-thread lock-step exchange (one host thread per leg-lane, spin barrier), so the
// kernel logic — per-leg dynamics, cross-leg reductions, PGS sweep order, ring bookkeeping — can be checked against
// the float64 oracle on a machine without a GPU.  It mirrors the b2q_* C ABI with host pointers.
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>
#include "../../paddlerobotics_b200/csrc/b2q_host_common.h"
#include "../gpu_probe/prim.h"

using namespace b2q;

namespace {

struct SpinBarrier {
  std::atomic<int> count{0};
  std::atomic<int> gen{0};
  void wait() {
    int g = gen.load(std::memory_order_acquire);
    if (count.fetch_add(1, std::memory_order_acq_rel) == 3) {
      count.store(0, std::memory_order_relaxed);
      gen.fetch_add(1, std::memory_order_release);
    } else {
      int spins = 0;
      while (gen.load(std::memory_order_acquire) == g) { if (++spins > 2000) { std::this_thread::yield(); spins = 0; } }
    }
  }
};
struct Exchange {
  SpinBarrier bar;
  alignas(64) volatile double A[4];
  alignas(64) volatile double Bf[4];
  alignas(64) double scr[SCRATCH_FLOATS];   // the robot's solver scratch (shared memory on the GPU)
};

template <typename T>
struct HostComm {
  int k; Exchange* x;
  int leg() const { return k; }
  template <typename U> U* scratch() const { return reinterpret_cast<U*>(x->scr); }
  void sync() const { x->bar.wait(); }
  bool any(bool f) const { return sum4(f ? T(1) : T(0)) > T(0); }
  T sum4(T v) const {  // same butterfly order as the shuffles: (v + v^1) + (that of lane^2)
    x->A[k] = (double)v; x->bar.wait();
    T p = v + (T)x->A[k ^ 1];
    x->Bf[k] = (double)p; x->bar.wait();
    T r = p + (T)x->Bf[k ^ 2];
    x->bar.wait();
    return r;
  }
  T bcast(T v, int f) const {
    x->A[k] = (double)v; x->bar.wait();
    T r = (T)x->A[f];
    x->bar.wait();
    return r;
  }
};

template <typename T>
struct Emu {
  B2QConfig cfg; Cfg<T> kc; Model<T> md; Buffers<T> B;
  std::vector<P4<T>> state, snap, snap_obs, param, etg, ring, pos_hist, extf; std::vector<int> step_count; std::vector<T> hf; std::vector<T> stage;
  int feat = 0;
  T def48[48];
  Exchange ex;
  template <class F>
  void run4(F f) {
    std::thread th[4];
    for (int k = 0; k < 4; k++) th[k] = std::thread([&, k]() { HostComm<T> cm{k, &ex}; f(cm); });
    for (auto& t : th) t.join();
  }
};

struct Handle { int prec; void* p; std::string err; };

template <typename T>
Emu<T>* create_t(const B2QConfig& c) {
  auto* e = new Emu<T>();
  e->cfg = c;
  int N = c.num_envs, Dm = c.ring_depth;
  if (c.terrain_type == 1) { e->hf.resize((size_t)c.hf_nx * c.hf_ny); for (size_t i = 0; i < e->hf.size(); i++) e->hf[i] = (T)c.hf_host[i]; }
  e->kc = make_cfg<T>(c, e->hf.empty() ? nullptr : e->hf.data());
  build_model_host(e->md, c.foot_radius, c.etg_T, c.etg_amp, c.etg_phase0, c.etg_phase1, c.etg_foot_y_inset);
  build_obs_map(e->md, c); e->feat = config_feat(c);
  e->pos_hist.assign((size_t)STUCK_H * N, P4<T>{0, 0, 0, 0}); e->extf.assign((size_t)N, P4<T>{0, 0, 0, 0}); e->stage.assign((size_t)N * OBS_DIM, T(0));
  e->state.assign((size_t)NS * N, P4<T>{0, 0, 0, 0}); e->snap = e->state;
  e->snap_obs.assign((size_t)12 * N, P4<T>{0, 0, 0, 0}); e->param.assign((size_t)NP * N, P4<T>{0, 0, 0, 0});
  e->etg.assign((size_t)NE * N, P4<T>{0, 0, 0, 0}); e->ring.assign((size_t)Dm * 2 * 12 * N, P4<T>{0, 0, 0, 0});
  e->step_count.assign(N, 0);
  double d48[48]; default_dyn_row(d48); for (int i = 0; i < 48; i++) e->def48[i] = (T)d48[i];
  e->B.N = N; e->B.Dm = Dm; e->B.state = e->state.data(); e->B.snap = e->snap.data(); e->B.snap_obs = e->snap_obs.data();
  e->B.param = e->param.data(); e->B.etg = e->etg.data(); e->B.ring = e->ring.data(); e->B.step_count = e->step_count.data();
  e->B.pos_hist = e->pos_hist.data(); e->B.extf = e->extf.data();
  return e;
}

template <typename T>
void set_dynamics_t(Emu<T>* e, const uint8_t* mask, const T* dyn) {
  int N = e->B.N;
  for (int i = 0; i < N; i++) if (!mask || mask[i]) pack_param_env<T>(dyn, e->def48, e->param.data(), N, i);
  e->run4([&](const HostComm<T>& cm) {
    for (int i = 0; i < N; i++) if (!mask || mask[i]) { if (e->feat) settle_lane<T, 1>(cm, e->kc, e->md, e->B, i, true); else settle_lane<T, 0>(cm, e->kc, e->md, e->B, i, true); }
  });
}
template <typename T>
void emit_rows(Emu<T>* e, const uint8_t* mask, T* obs) {
  const int od = e->md.obs_dim;
  for (int i = 0; i < e->B.N; i++) if (!mask || mask[i]) for (int j = 0; j < od; j++) obs[(size_t)i * od + j] = obs_out_elem(e->md, e->stage.data() + (size_t)i * OBS_DIM, j);
}
template <typename T>
void reset_t(Emu<T>* e, const uint8_t* mask, const T* w, const T* b, const T* xoff, T* obs) {
  int N = e->B.N;
  for (int i = 0; i < N; i++) if (!mask || mask[i]) pack_etg_env<T>(w, b, e->etg.data(), N, i);
  e->run4([&](const HostComm<T>& cm) { for (int i = 0; i < N; i++) if (!mask || mask[i]) reset_lane(cm, e->kc, e->md, e->B, i, true, e->stage.data() + (size_t)i * OBS_DIM, xoff); });
  if (obs) emit_rows(e, mask, obs);
}
template <typename T>
void step_t(Emu<T>* e, const T* action, int donef, T* obs, T* rew, uint8_t* done, T* info) {
  int N = e->B.N;
  e->run4([&](const HostComm<T>& cm) {
    for (int i = 0; i < N; i++) {
      if (e->feat) step_lane<T, 1>(cm, e->kc, e->md, e->B, i, true, action, donef, e->cfg.auto_reset, e->stage.data(), rew, done, info);
      else step_lane<T, 0>(cm, e->kc, e->md, e->B, i, true, action, donef, e->cfg.auto_reset, e->stage.data(), rew, done, info);
    }
  });
  emit_rows<T>(e, nullptr, obs);
}
template <typename T>
void set_force_t(Emu<T>* e, const T* f) {
  for (int i = 0; i < e->B.N; i++) e->extf[i] = f ? P4<T>{f[3 * i], f[3 * i + 1], f[3 * i + 2], T(0)} : P4<T>{0, 0, 0, 0};
}

}  // namespace

extern "C" {
void emu_default_config(B2QConfig* c) { default_config(c); }
int emu_create(const B2QConfig* c, void** out) {
  if (!c || !out || validate_config(*c)) return B2Q_EINVAL;
  auto* h = new Handle();
  h->prec = c->precision;
  h->p = c->precision ? (void*)create_t<double>(*c) : (void*)create_t<float>(*c);
  *out = h;
  if (c->precision) set_dynamics_t<double>((Emu<double>*)h->p, nullptr, nullptr); else set_dynamics_t<float>((Emu<float>*)h->p, nullptr, nullptr);
  return B2Q_OK;
}
int emu_destroy(void* hv) { auto* h = (Handle*)hv; if (h->prec) delete (Emu<double>*)h->p; else delete (Emu<float>*)h->p; delete h; return 0; }
int emu_set_dynamics(void* hv, const uint8_t* mask, const void* dyn) {
  auto* h = (Handle*)hv;
  if (h->prec) set_dynamics_t<double>((Emu<double>*)h->p, mask, (const double*)dyn); else set_dynamics_t<float>((Emu<float>*)h->p, mask, (const float*)dyn);
  return 0;
}
int emu_reset(void* hv, const uint8_t* mask, const void* w, const void* b, const void* xoff, void* obs) {
  auto* h = (Handle*)hv;
  if (h->prec) reset_t<double>((Emu<double>*)h->p, mask, (const double*)w, (const double*)b, (const double*)xoff, (double*)obs);
  else reset_t<float>((Emu<float>*)h->p, mask, (const float*)w, (const float*)b, (const float*)xoff, (float*)obs);
  return 0;
}
int emu_set_force(void* hv, const void* f) {
  auto* h = (Handle*)hv;
  if (h->prec) set_force_t<double>((Emu<double>*)h->p, (const double*)f); else set_force_t<float>((Emu<float>*)h->p, (const float*)f);
  return 0;
}
int emu_obs_dim(void* hv) { auto* h = (Handle*)hv; return h->prec ? ((Emu<double>*)h->p)->md.obs_dim : ((Emu<float>*)h->p)->md.obs_dim; }
int emu_step(void* hv, const void* action, int donef, void* obs, void* rew, uint8_t* done, void* info) {
  auto* h = (Handle*)hv;
  if (h->prec) step_t<double>((Emu<double>*)h->p, (const double*)action, donef, (double*)obs, (double*)rew, done, (double*)info);
  else step_t<float>((Emu<float>*)h->p, (const float*)action, donef, (float*)obs, (float*)rew, done, (float*)info);
  return 0;
}
int emu_get_state(void* hv, void* out) {
  auto* h = (Handle*)hv;
  if (h->prec) { auto* e = (Emu<double>*)h->p; for (int i = 0; i < e->B.N; i++) get_state_env<double>(e->state.data(), (double*)out, e->B.N, i); }
  else { auto* e = (Emu<float>*)h->p; for (int i = 0; i < e->B.N; i++) get_state_env<float>(e->state.data(), (float*)out, e->B.N, i); }
  return 0;
}
int emu_set_state(void* hv, const void* in) {
  auto* h = (Handle*)hv;
  if (h->prec) { auto* e = (Emu<double>*)h->p; for (int i = 0; i < e->B.N; i++) set_state_env<double>(e->state.data(), (const double*)in, e->B.N, i); }
  else { auto* e = (Emu<float>*)h->p; for (int i = 0; i < e->B.N; i++) set_state_env<float>(e->state.data(), (const float*)in, e->B.N, i); }
  return 0;
}

// ---- the scalar primitives through their host branches, one element at a time (tests/gpu_probe/prim.h; the probe runs the device ones)
void emu_sincos_f(int n, const float* a, float* s, float* c) { for (int i = 0; i < n; i++) b2q_prim::sincos_f(a[i], s + i, c + i); }
void emu_unary_f(int which, int n, const float* x, float* y) { for (int i = 0; i < n; i++) y[i] = which == 0 ? b2q_prim::rcp_f(x[i]) : b2q_prim::rsqrt_f(x[i]); }
void emu_philox4(int n, const uint64_t* seed, const uint32_t* ctr, uint32_t* out) {
  for (int i = 0; i < n; i++) philox4(seed[i], ctr[3 * i], ctr[3 * i + 1], ctr[3 * i + 2], out + 4 * i);
}
void emu_philox_normal4(int prec, int n, const uint64_t* seed, const uint32_t* ctr, void* out) {
  for (int i = 0; i < n; i++) {
    if (prec) philox_normal4<double>(seed[i], ctr[3 * i], ctr[3 * i + 1], ctr[3 * i + 2], (double*)out + 4 * i);
    else philox_normal4<float>(seed[i], ctr[3 * i], ctr[3 * i + 1], ctr[3 * i + 2], (float*)out + 4 * i);
  }
}
void emu_leg(int prec, int n, int inverse, const int* leg, const void* in, void* out) {
  if (prec) {
    Model<double> md = b2q_prim::default_model<double>(); const double* x = (const double*)in; double* y = (double*)out;
    for (int i = 0; i < n; i++) if (leg[i] >= 0 && leg[i] < 4) { if (inverse) b2q_prim::leg_inv(md, leg[i], x + 3 * i, y + 3 * i); else b2q_prim::leg_fk(md, leg[i], x + 3 * i, y + 3 * i); }
  } else {
    Model<float> md = b2q_prim::default_model<float>(); const float* x = (const float*)in; float* y = (float*)out;
    for (int i = 0; i < n; i++) if (leg[i] >= 0 && leg[i] < 4) { if (inverse) b2q_prim::leg_inv(md, leg[i], x + 3 * i, y + 3 * i); else b2q_prim::leg_fk(md, leg[i], x + 3 * i, y + 3 * i); }
  }
}
void emu_rpy(int prec, int n, const void* q, void* out) {
  for (int i = 0; i < n; i++) {
    if (prec) b2q_prim::rpy((const double*)q + 4 * i, (double*)out + 3 * i); else b2q_prim::rpy((const float*)q + 4 * i, (float*)out + 3 * i);
  }
}
void emu_terrain(int prec, int nx, int ny, double x0, double y0, double cell, const double* hf, int n, const void* xy, void* out) {
  if (prec) {
    std::vector<double> h(hf, hf + (size_t)nx * ny); Cfg<double> cf = b2q_prim::hf_cfg<double>(nx, ny, x0, y0, cell, h.data());
    for (int i = 0; i < n; i++) b2q_prim::terrain(cf, ((const double*)xy)[2 * i], ((const double*)xy)[2 * i + 1], (double*)out + 4 * i);
  } else {
    std::vector<float> h(hf, hf + (size_t)nx * ny); Cfg<float> cf = b2q_prim::hf_cfg<float>(nx, ny, x0, y0, cell, h.data());
    for (int i = 0; i < n; i++) b2q_prim::terrain(cf, ((const float*)xy)[2 * i], ((const float*)xy)[2 * i + 1], (float*)out + 4 * i);
  }
}
void emu_solve(int prec, int n, const void* S, const void* b, void* x) {
  for (int i = 0; i < n; i++) {
    if (prec) b2q_prim::spd_solve((const double*)S + 21 * i, (const double*)b + 6 * i, (double*)x + 6 * i);
    else b2q_prim::spd_solve((const float*)S + 21 * i, (const float*)b + 6 * i, (float*)x + 6 * i);
  }
}
}
