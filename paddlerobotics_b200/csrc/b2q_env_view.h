// b2q_env_view.h — what kernels outside b2q_api.cu (b2q_deploy.cu) may see of an env handle: sizes, element type and the device
// buffers they read.  Defined in b2q_api.cu, where the handle's type lives.
#pragma once
#include <stdint.h>
#include "../../include/b2q.h"

namespace b2q {

struct EnvView {
  int N, obs_dim, elem_size, device, etg_enabled;
  const int32_t* step_count;   // [N] device: control steps since each env's reset (the step kernel's B.step_count)
  const void* model;           // device Model<T> (T = float for elem_size 4, double for 8)
  const void* state;           // device P4<T> state packs [NS][N]; packs 4..7 hold the joint angles of legs 0..3 in x, y, z
};

// B2Q_EINVAL for a NULL handle
int env_view(B2QHandle h, EnvView* v);
// sets the message b2q_last_error(h) returns
void env_set_error(B2QHandle h, const char* msg);

}  // namespace b2q
