// b2q_mlp_internal.h — library-internal extension of the MLP forward used by the SAC trainer (b2q_sac.cu): the same
// fused wgmma kernel, additionally dumping the bf16 layer inputs it already holds in shared memory, in the two layouts
// the backward GEMMs consume ([batch x width] and [width x batch]).  Not part of the public C ABI.
#pragma once
#include <cuda_bf16.h>
#include <cstdint>
#include "../../include/b2q_mlp.h"

struct B2QMlpSaves {
  __nv_bfloat16* x_rm;   // [M][64]            concatenated, zero-padded input
  __nv_bfloat16* x_t;    // [64][M]
  __nv_bfloat16* h1_rm;  // [nets][M][256]     relu(layer 1)
  __nv_bfloat16* h1_t;   // [nets][256][M]
  __nv_bfloat16* h2_rm;  // [nets][M][256]     relu(layer 2)
  __nv_bfloat16* h2_t;   // [nets][256][M]
};
// `seed_ctr` (optional): device-side counter folded into the sampling key when eps == NULL (b2q_philox.cuh), for CUDA-graph replays.
// `da` (optional, out_dim == 1 nets): f32 [nets][M][16] — the gradient of each net's output wrt the action columns of its input, computed in the
// same kernel right after the forward (dh2 = W3 . relu'(h2), dh1 = (dh2 W2) . relu'(h1), da = dh1 W1[:, action]), activations never leaving the SM
extern "C" int b2q_mlp_forward_ex(B2QMlpHandle h, const float* in1, int in1_dim, const float* in2, int M, int mode, uint64_t seed, const float* eps,
                                  float* out, float* logp, float* raw, const B2QMlpSaves* saves, float* da, const int* seed_ctr, void* stream);

// Layout of one net's forward image in HBM (bf16 K-major SWIZZLE_128B operand images + f32 biases [b1 | b2 | b3 padded to 32]); the SAC
// optimiser kernels write updated parameters straight into it (b2q_sac.cu: k_adam_pack / k_polyak_pack).
namespace b2q_mlp_img {
constexpr size_t SZ_W1 = 32768, SZ_W2 = 131072, SZ_W3 = 16384, SZ_BIAS = (B2Q_MLP_HIDDEN + B2Q_MLP_HIDDEN + 32) * 4;
constexpr size_t IMG_W1 = 0, IMG_W2 = SZ_W1, IMG_W3 = IMG_W2 + SZ_W2, IMG_BIAS = IMG_W3 + SZ_W3;
// operand images of the input-gradient pass (forward_ex with `da`): W2^T as the B operand of dh1 = dh2 W2 ([N = in][K = out]) and the action
// columns of W1 ([N = 16 action slots][K = 256 hidden]) for da = dh1 W1[:, a_off : a_off + a_dim]
constexpr size_t SZ_W2T = SZ_W2, SZ_W1A = 16 * B2Q_MLP_HIDDEN * 2;
constexpr size_t IMG_W2T = IMG_BIAS + SZ_BIAS, IMG_W1A = IMG_W2T + SZ_W2T, IMG_BYTES = IMG_W1A + SZ_W1A;
static_assert(IMG_W2T % 16 == 0 && IMG_W1A % 16 == 0 && IMG_BYTES % 16 == 0, "bulk copies need 16-byte aligned sources");
}
// which input columns are the action (critic nets): selects the W1 columns packed into the W1A image.  Default: none (image stays zero).
extern "C" int b2q_mlp_set_action_slice(B2QMlpHandle h, int a_off, int a_dim);
extern "C" uint8_t* b2q_mlp_image(B2QMlpHandle h, int net);   // device pointer of net's image (library-internal)
