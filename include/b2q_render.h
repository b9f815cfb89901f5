/* b2q_render.h — camera images of the batched A1 simulator: a ray-cast counterpart of pybullet's getCameraImage
 * (ETGRL/train.py:197, BCtrain.py:163: p.getCameraImage(640, 480, ...)[2] written to img/img{step}.jpg).
 *
 * Device pointers, the caller's stream, no host synchronisation; 0 on success, a negative B2Q_E* code otherwise with the
 * message in b2q_last_error(h).
 *
 * The caller passes the state rows to draw, [N,37] in the handle's precision exactly as b2q_get_state writes them
 * (pos3 quat4(xyzw) vlin3 vang3 q12 qd12): the live batch, a recorded trajectory or any other state.  The handle supplies the
 * model constants and its terrain (the plane z = 0 or its height field, including the edge-clamped extension outside the grid).
 * View v draws the robot of row env_ids[v] through the camera view[v], proj[v].
 *
 * Camera conventions are pybullet's: view and proj are column-major 4x4 OpenGL matrices (computeViewMatrix,
 * computeProjectionMatrixFOV; orthographic projections work too).  Row 0 of an image is its top row and each pixel is sampled
 * at its centre.  All math is float32 for both handle precisions.
 *   rgba  [V,H,W,4] uint8, alpha 255; Lambert shading from one directional light, a fixed colour per segmentation class,
 *         a 0.25 m checkerboard on the terrain, sky colour on a miss
 *   depth [V,H,W] float32, the OpenGL depth-buffer value in [0,1]; linear depth = far*near/(far-(far-near)*depth); a miss is 1
 *   seg   [V,H,W] int32 segmentation ids (this project's own; the URDF link indices are not available):
 *           -1 sky, 0 terrain, 1 trunk, 2 + 4*leg + {0 hip, 1 thigh, 2 calf, 3 toe}  (legs 0 FR, 1 FL, 2 RR, 3 RL)
 * Any of rgba, depth, seg may be NULL; rgba must be 4-byte aligned.
 *
 * A state row with a non-finite value renders without the robot; a camera with a non-finite or singular proj*view renders
 * the miss values; an env_id outside [0, N) fills its view with the miss values and reads no state.
 * B2Q_EINVAL: V < 1 or V > 65535, width or height < 1, NULL state / env_ids / view / proj.
 *
 * Collision geometry drawn (unverified, see DESIGN.md "Camera images"): trunk box 0.267 x 0.194 x 0.114 m, hip cylinders
 * r 0.046 m x 0.04 m, thigh boxes 0.034 x 0.0245 x 0.2 m, calf boxes 0.016 x 0.016 x 0.2 m, toe spheres of foot_radius.
 */
#ifndef B2Q_RENDER_H
#define B2Q_RENDER_H
#include <stdint.h>
#include "b2q.h"
#ifdef __cplusplus
extern "C" {
#endif

int b2q_render(B2QHandle h, const void* state /*[N,37]*/, const int32_t* env_ids /*[V]*/, int V, const float* view /*[V,16]*/,
               const float* proj /*[V,16]*/, int width, int height, uint8_t* rgba /*[V,H,W,4] or NULL*/, float* depth /*[V,H,W] or NULL*/,
               int32_t* seg /*[V,H,W] or NULL*/, void* stream);

#ifdef __cplusplus
}
#endif
#endif
