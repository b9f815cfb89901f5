// b2q_mlp_internal.h — library-internal parts of the MLP that the SAC trainer (b2q_sac.cu) shares: the forward extension (the same
// fused wgmma kernel, additionally dumping the bf16 layer inputs it already holds in shared memory, in the two layouts the backward
// GEMMs consume: [batch x width] and [width x batch]) and the packer that writes the weight images.  Not part of the public C ABI.
#pragma once
#include <cuda_bf16.h>
#include <cstdint>
#include "../../include/b2q_mlp.h"
#include "b2q_tc.cuh"

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

// Layout of one net's forward image in HBM (bf16 K-major SWIZZLE_128B operand images + f32 biases [b1 | b2 | b3 padded to 32]).
namespace b2q_mlp_img {
constexpr size_t SZ_W1 = 32768, SZ_W2 = 131072, SZ_W3 = 16384, SZ_BIAS = (B2Q_MLP_HIDDEN + B2Q_MLP_HIDDEN + 32) * 4;
constexpr size_t IMG_W1 = 0, IMG_W2 = SZ_W1, IMG_W3 = IMG_W2 + SZ_W2, IMG_BIAS = IMG_W3 + SZ_W3;
// operand images of the input-gradient pass (forward_ex with `da`): W2^T as the B operand of dh1 = dh2 W2 ([N = in][K = out]) and the action
// columns of W1 ([N = 16 action slots][K = 256 hidden]) for da = dh1 W1[:, a_off : a_off + a_dim]
constexpr size_t SZ_W2T = SZ_W2, SZ_W1A = 16 * B2Q_MLP_HIDDEN * 2;
constexpr size_t IMG_W2T = IMG_BIAS + SZ_BIAS, IMG_W1A = IMG_W2T + SZ_W2T, IMG_BYTES = IMG_W1A + SZ_W1A;
static_assert(IMG_W2T % 16 == 0 && IMG_W1A % 16 == 0 && IMG_BYTES % 16 == 0, "bulk copies need 16-byte aligned sources");
}

// Where each parameter of one net lands: its forward image and, for the SAC learner's nets, the bf16 copies the backward GEMMs read
// (W2^T [256][256], W3^T [256][64], the action columns of W1 [16][256]; null for nets without a backward pass).  Parameter i is the
// i-th float of the flat [W1 | b1 | W2 | b2 | W3 | b3] (nn.Linear [out][in] weights).  Only real entries are written: the padding of the
// images and copies (W1 columns >= in_dim, W3 rows >= od, W1A rows >= a_dim) is zero from the memset at allocation and nothing ever
// writes it.  The W2^T / W1A images are written only with `gradin` (a_dim > 0): their one reader, forward_ex with `da`, rejects a_dim < 1.
struct PackDst { uint8_t* img; __nv_bfloat16 *W2T, *W3T, *W1A; int in_dim, od, a_off, a_dim, gradin; unsigned oW1, ob1, oW2, ob2, oW3, ob3, n; };
struct PackDst2 { PackDst d[2]; };   // two nets of one handle, parameter blocks of d[0].n floats back to back
// a net's destinations without backward copies
inline PackDst pack_dst(uint8_t* img, int in_dim, int od, int a_off, int a_dim) {
  constexpr unsigned H = B2Q_MLP_HIDDEN;
  PackDst d{img, nullptr, nullptr, nullptr, in_dim, od, a_off, a_dim, a_dim > 0 ? 1 : 0};
  d.oW1 = 0; d.ob1 = H * (unsigned)in_dim; d.oW2 = d.ob1 + H; d.ob2 = d.oW2 + H * H; d.oW3 = d.ob2 + H; d.ob3 = d.oW3 + (unsigned)od * H; d.n = d.ob3 + (unsigned)od;
  return d;
}
// the only code that maps (net, parameter index) to image bytes and backward-copy elements: b2q_mlp_set_weights and the SAC learner's
// Adam / Polyak / pack kernels (b2q_sac.cu) all store through it
__device__ __forceinline__ void pack_param(const PackDst& d, unsigned i, float v) {
  using b2q_tc::sw128_offset;
  constexpr int H = B2Q_MLP_HIDDEN;
  const __nv_bfloat16 vb = __float2bfloat16(v);
  float* bias = reinterpret_cast<float*>(d.img + b2q_mlp_img::IMG_BIAS);
  if (i < d.ob1) {                                   // W1 [256][in_dim]
    const int n = (int)(i / (unsigned)d.in_dim), k = (int)i - n * d.in_dim;
    *reinterpret_cast<__nv_bfloat16*>(d.img + b2q_mlp_img::IMG_W1 + sw128_offset(n, k, H)) = vb;
    if (k >= d.a_off && k < d.a_off + d.a_dim) {
      if (d.W1A) d.W1A[(size_t)(k - d.a_off) * H + n] = vb;
      if (d.gradin) *reinterpret_cast<__nv_bfloat16*>(d.img + b2q_mlp_img::IMG_W1A + sw128_offset(k - d.a_off, n, 16)) = vb;
    }
  } else if (i < d.oW2) { bias[i - d.ob1] = v;
  } else if (i < d.ob2) {                            // W2 [256][256]
    const int j = (int)(i - d.oW2), n = j >> 8, k = j & 255;
    *reinterpret_cast<__nv_bfloat16*>(d.img + b2q_mlp_img::IMG_W2 + sw128_offset(n, k, H)) = vb;
    if (d.W2T) d.W2T[(size_t)k * H + n] = vb;
    if (d.gradin) *reinterpret_cast<__nv_bfloat16*>(d.img + b2q_mlp_img::IMG_W2T + sw128_offset(k, n, H)) = vb;
  } else if (i < d.oW3) { bias[H + i - d.ob2] = v;
  } else if (i < d.ob3) {                            // W3 [od][256]
    const int j = (int)(i - d.oW3), n = j >> 8, k = j & 255;
    *reinterpret_cast<__nv_bfloat16*>(d.img + b2q_mlp_img::IMG_W3 + sw128_offset(n, k, 32)) = vb;
    if (d.W3T) d.W3T[(size_t)k * 64 + n] = vb;
  } else { bias[2 * H + i - d.ob3] = v; }
}

// which input columns are the action (critic nets): selects the W1 columns packed into the W1A image.  Default: none (image stays zero).
// Set it before the weights: b2q_mlp_set_weights writes only the columns of the current slice.
extern "C" int b2q_mlp_set_action_slice(B2QMlpHandle h, int a_off, int a_dim);
extern "C" uint8_t* b2q_mlp_image(B2QMlpHandle h, int net);   // device pointer of net's image (library-internal)
