// b2q_render_internal.h — the launcher of the camera-image kernel (b2q_render.cu), called by b2q_api.cu after it has validated
// the arguments of b2q_render (include/b2q_render.h).
#pragma once
#include <cuda_runtime.h>
#include "b2q_render.cuh"

namespace b2q {

template <typename T>
struct RenderArgs {
  Model<float> md;          // model constants in float32 (leg_kin inputs, foot radius)
  RTerrain tr;
  const T* hf;              // the handle's device height field [ny][nx] (type 1)
  const T* state;           // [N][37]
  int N;
  const int32_t* env_ids;   // [V]
  const float* view;        // [V][16]
  const float* proj;        // [V][16]
  int W, H;
  uint8_t* rgba;            // [V][H][W][4] or null
  float* depth;             // [V][H][W] or null
  int32_t* seg;             // [V][H][W] or null
};

template <typename T>
cudaError_t render_launch(const RenderArgs<T>& a, int V, cudaStream_t s);

}  // namespace b2q
