// emu_render.cpp — CPU build of the camera-image device code in paddlerobotics_b200/csrc/b2q_render.cuh.
//
// TEST INFRASTRUCTURE ONLY (tests/emu/render.mk -> libb2q_emu_render.so in a directory the tests choose).  It compiles the very same scene, camera
// and per-pixel functions the sm_90a kernel calls, with the scene built serially instead of one thread per leg, so the ray-caster
// can be checked against the NumPy reference (tests/render_ref.py) on a machine without a GPU.  Height field and state in float64,
// as a float64 handle passes them.
#include <cstring>
#include "../../paddlerobotics_b200/csrc/b2q_render.cuh"
#include "../../paddlerobotics_b200/csrc/b2q_model_host.h"

using namespace b2q;

extern "C" {
// state [37]; hf [ny][nx] or null (plane); view / proj [16] column-major; rgba [H][W][4], depth [H][W], seg [H][W].
int emu_render(const double* state, double foot_radius, const double* hf, int nx, int ny, double x0, double y0, double cell, const float* view,
               const float* proj, int W, int H, unsigned char* rgba, float* depth, int* seg) {
  Model<float> md;
  build_model_host(md, foot_radius, 0.5, 0.2, -3.14159265358979323846 / 2, 0.0);
  RScene sc;
  std::memset(&sc, 0, sizeof sc);
  if (state) {
    float st[37];
    for (int i = 0; i < 37; i++) st[i] = (float)state[i];
    render_scene(md, st, sc);
  }
  RCam cam;
  render_camera(view, proj, cam);
  RTerrain tr;
  std::memset(&tr, 0, sizeof tr);
  if (hf) {
    tr.type = 1; tr.nx = nx; tr.ny = ny; tr.x0 = (float)x0; tr.y0 = (float)y0; tr.icell = (float)(1.0 / cell);
    tr.lo = tr.hi = (float)hf[0];
    for (int i = 0; i < nx * ny; i++) { tr.lo = std::fmin(tr.lo, (float)hf[i]); tr.hi = std::fmax(tr.hi, (float)hf[i]); }
  }
  for (int py = 0; py < H; py++)
    for (int px = 0; px < W; px++) {
      const size_t i = (size_t)py * W + px;
      render_pixel<double>(sc, cam, tr, hf, px, py, W, H, rgba + 4 * i, depth[i], seg[i]);
    }
  return 0;
}
}
