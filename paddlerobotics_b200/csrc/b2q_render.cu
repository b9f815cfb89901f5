// b2q_render.cu — sm_90a camera-image kernel (include/b2q_render.h): one CTA per (view, 16 x 16 pixel tile), one thread per pixel.
// The CTA's prologue builds the view's camera (proj * view and its inverse) and its 17 primitives (one thread per leg, leg_kin()
// in float32) in shared memory; every thread then casts the ray through its pixel centre (b2q_render.cuh).
#include "b2q_render_internal.h"

namespace b2q {
namespace {

template <typename T>
__global__ void __launch_bounds__(RENDER_TILE * RENDER_TILE) b2q_render_kernel(const __grid_constant__ RenderArgs<T> a) {
  __shared__ RScene sc;
  __shared__ RCam cam;
  __shared__ float st[37];
  const int v = blockIdx.y;
  const int tid = threadIdx.x + RENDER_TILE * threadIdx.y;
  const int env = a.env_ids[v];
  const bool env_ok = env >= 0 && env < a.N;
  if (tid < 37) st[tid] = env_ok ? (float)a.state[(size_t)env * 37 + tid] : 0.0f;
  if (tid == 64) {
    float vm[16], pm[16];
    for (int i = 0; i < 16; i++) { vm[i] = a.view[(size_t)v * 16 + i]; pm[i] = a.proj[(size_t)v * 16 + i]; }
    render_camera(vm, pm, cam);
    if (!env_ok) cam.ok = 0;   // an env id outside [0, N): the whole view is the miss values
  }
  const int bad = __syncthreads_or(tid < 37 && !r_finite(st[tid]));
  if (tid == 0) sc.robot = bad ? 0 : 1;
  if (!bad) {
    if (tid < 4) render_leg(a.md, tid, st, sc.p + 1 + 4 * tid);
    else if (tid == 4) render_trunk(st, sc.p[0]);
  }
  __syncthreads();
  if (tid == 0 && !bad) render_bound(sc);
  __syncthreads();
  const int tiles_x = (a.W + RENDER_TILE - 1) / RENDER_TILE;
  const int px = (blockIdx.x % tiles_x) * RENDER_TILE + threadIdx.x, py = (blockIdx.x / tiles_x) * RENDER_TILE + threadIdx.y;
  if (px >= a.W || py >= a.H) return;
  unsigned char c[4]; float d; int s;
  render_pixel<T>(sc, cam, a.tr, a.hf, px, py, a.W, a.H, c, d, s);
  const size_t i = ((size_t)v * a.H + py) * a.W + px;   // 64-bit: V * H * W * 4 bytes passes 2^31 at sizes users ask for
  if (a.rgba) reinterpret_cast<uchar4*>(a.rgba)[i] = make_uchar4(c[0], c[1], c[2], c[3]);
  if (a.depth) a.depth[i] = d;
  if (a.seg) a.seg[i] = s;
}

}  // namespace

template <typename T>
cudaError_t render_launch(const RenderArgs<T>& a, int V, cudaStream_t s) {
  const dim3 grid((unsigned)(((a.W + RENDER_TILE - 1) / RENDER_TILE) * ((a.H + RENDER_TILE - 1) / RENDER_TILE)), (unsigned)V);
  b2q_render_kernel<T><<<grid, dim3(RENDER_TILE, RENDER_TILE), 0, s>>>(a);
  return cudaGetLastError();
}
template cudaError_t render_launch<float>(const RenderArgs<float>&, int, cudaStream_t);
template cudaError_t render_launch<double>(const RenderArgs<double>&, int, cudaStream_t);

}  // namespace b2q
