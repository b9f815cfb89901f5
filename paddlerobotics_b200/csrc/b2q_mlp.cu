// b2q_mlp.cu — K3: fused 3-layer MLP forward (in<=64 -> 256 -> 256 -> out<=32) on Hopper warpgroup MMAs (wgmma).
//
// One CTA (256 threads = two warpgroups, each owning 64 rows of the tile in its MMAs) per 128-row tile of the batch:
//   * weights live in HBM as ready-made shared-memory images (bf16, K-major, 128-byte swizzle, 64-column panels) and are
//     brought in by bulk async copies (cp.async.bulk) that complete on mbarriers;
//   * the input tile is converted f32 -> bf16 by the CTA's threads straight into the swizzled A-operand layout;
//   * each layer is a chain of wgmma.mma_async (M=64 per warpgroup, N=256|32, K=16) with both operands in shared memory,
//     accumulating in registers (128 f32 per thread for N=256);
//   * the epilogue applies bias+ReLU in f32 to the accumulator fragment and writes the bf16 activations back into the A-operand
//     region for the next layer, so activations never leave the SM; the last epilogue applies tanh / clamp / sampling /
//     log-prob and stores f32.
// Shared memory: A 64 KB | W2 128 KB | W1 then W3 32 KB | biases 2.1 KB | barriers  = 226.2 KB (of 227 KB).
// Reference: Actor/Critic.forward (model/mujoco_model.py:44-89), SAC.predict/sample (alg/sac.py:60-75).
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <new>
#include <string>
#include "../../include/b2q_mlp.h"
#include "b2q_tc.cuh"
#include "b2q_mlp_internal.h"
#include "b2q_philox.cuh"

using namespace b2q_tc;

namespace {

constexpr int HID = B2Q_MLP_HIDDEN;
constexpr int TILE_M = 128;
using b2q_mlp_img::IMG_W1; using b2q_mlp_img::IMG_W2; using b2q_mlp_img::IMG_W3; using b2q_mlp_img::IMG_BIAS; using b2q_mlp_img::IMG_BYTES;
using b2q_mlp_img::IMG_W2T; using b2q_mlp_img::IMG_W1A;
constexpr uint32_t SZ_W1A = (uint32_t)b2q_mlp_img::SZ_W1A, OFF_W1A_IN_W13 = 16384;   // the W1A image sits behind W3 in the (32 KB) W1/W3 region
constexpr uint32_t SZ_A = 65536, SZ_W2 = (uint32_t)b2q_mlp_img::SZ_W2, SZ_W13 = 32768, SZ_W1 = (uint32_t)b2q_mlp_img::SZ_W1, SZ_W3 = (uint32_t)b2q_mlp_img::SZ_W3,
                   SZ_BIAS = (uint32_t)b2q_mlp_img::SZ_BIAS;
constexpr uint32_t OFF_A = 0, OFF_W2 = OFF_A + SZ_A, OFF_W13 = OFF_W2 + SZ_W2, OFF_BIAS = OFF_W13 + SZ_W13, OFF_BAR = OFF_BIAS + SZ_BIAS;
constexpr uint32_t SMEM_BYTES = OFF_BAR + 64 + 512;   // + the head's log-prob exchange [128] f32
static_assert(SMEM_BYTES <= 232448, "exceeds 227 KB of shared memory per CTA");

using b2q_philox::philox_normal;

struct FwdArgs {
  const float* in1; const float* in2; int in1_dim, in_dim, out_dim, M, mode; uint64_t seed; const float* eps;
  float* out; float* logp; float* raw; const uint8_t* img; size_t img_stride;
  B2QMlpSaves sv; int save;
  float* da;   // input-gradient pass (see b2q_mlp_internal.h) or null
  const int* seed_ctr;   // device-side counter folded into the sampling key (b2q_philox.cuh) or null
};

// actor head of one row, actions j with (j & 1) == chalf: tanh(mean) or the rsample() + tanh-Gaussian log-prob; returns the row's log-prob share.
// AC > 0: the action dimension as a compile-time constant (the TMEM register array stays statically indexed); AC == 0: runtime dimension.
template <int AC>
__device__ __forceinline__ float head_actions(const uint32_t (&r)[32], const float* b3, const FwdArgs& a, int row, size_t orow, int chalf) {
  const int A = AC > 0 ? AC : (a.out_dim >> 1);
  const uint64_t seed_eff = b2q_philox::effective_seed(a.seed, a.seed_ctr);
  float y[32];
#pragma unroll
  for (int j = 0; j < 32; j++) y[j] = __uint_as_float(r[j]) + b3[j];
  float lp = 0.f;
#pragma unroll
  for (int j = 0; j < (AC > 0 ? AC : 16); j++) {
    if ((j & 1) != chalf || j >= A) continue;
    const float mean = y[j];
    float act;
    if (a.mode == B2Q_MLP_PREDICT) {
      act = tanhf(mean);                                                   // sac.py:60-63
    } else {
      const float ls = fminf(fmaxf(y[A + j], -20.f), 2.f), sd = expf(ls);  // mujoco_model.py:21-22,59
      const float e = a.eps ? a.eps[(size_t)row * A + j] : philox_normal(seed_eff, (uint32_t)row, (uint32_t)j);
      const float x = mean + sd * e;                                       // rsample
      act = tanhf(x);
      lp += -0.5f * e * e - ls - 0.9189385332046727f;                      // Normal.log_prob(x)
      lp -= logf((1.f - act * act) + 1e-6f);                               // sac.py:72
    }
    a.out[orow * A + j] = act;
  }
  return lp;
}

constexpr int NTHR = 256;
__global__ void __launch_bounds__(NTHR, 1) b2q_mlp_fwd_kernel(FwdArgs a) { pdl_sync();
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, net = blockIdx.y;
  const int trow = tid & (TILE_M - 1), chalf = tid >> 7;   // row-wise passes: tile row owned; column half (0: cols 0..127, 1: 128..255)
  const int wg = tid >> 7;                                 // warpgroup: MMA rows 64 wg .. 64 wg + 63 of the tile
  const int fr0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), fc0 = 2 * (lane & 3);   // accumulator fragment: rows fr0, fr0 + 8; columns 8 j + fc0 + {0, 1}
  const int row0 = blockIdx.x * TILE_M, row = row0 + trow;
  const uint32_t sbase = smem_u32(smem);
  if ((sbase & 1023u) != 0) __trap();   // SWIZZLE_128B operands need a 1024-byte aligned base
  const uint32_t sA = sbase + OFF_A, sAw = sA + (uint32_t)wg * 64u * 128u, sW2 = sbase + OFF_W2, sW13 = sbase + OFF_W13;
  const uint32_t bar_w1 = sbase + OFF_BAR, bar_w2 = bar_w1 + 8, bar_w3 = bar_w1 + 16, bar_w2t = bar_w1 + 32;
  const float* bias = reinterpret_cast<const float*>(smem + OFF_BIAS);
  const uint8_t* img = a.img + (size_t)net * a.img_stride;

  if (tid == 0) {
    mbar_init(bar_w1, 1); mbar_init(bar_w2, 1); mbar_init(bar_w3, 1); mbar_init(bar_w2t, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // weights: W1 (+biases) first, then W2 in 32 KB pieces
    mbar_expect_tx(bar_w1, SZ_W1 + SZ_BIAS);
    bulk_g2s(sW13, img + IMG_W1, SZ_W1, bar_w1);
    bulk_g2s(sbase + OFF_BIAS, img + IMG_BIAS, SZ_BIAS, bar_w1);
    mbar_expect_tx(bar_w2, SZ_W2);
#pragma unroll
    for (int i = 0; i < 4; i++) bulk_g2s(sW2 + i * 32768u, img + IMG_W2 + (size_t)i * 32768u, 32768u, bar_w2);
  }
  // input tile: f32 [rows, in_dim] (two sources concatenated) -> bf16 swizzled panel 0 (K padded to 64 with zeros)
  {
    const int in2_dim = a.in_dim - a.in1_dim;
    // 32 elements per thread (one column k = tid & 63, rows (tid >> 6) + 4 j), ALL loads in flight before the first use
    constexpr int PER = 64 * TILE_M / NTHR;
    const int k = tid & 63;
    const float* src = k < a.in1_dim ? a.in1 + k : (k < a.in_dim ? a.in2 + (k - a.in1_dim) : nullptr);
    const int ld = k < a.in1_dim ? a.in1_dim : in2_dim;
    float v[PER];
#pragma unroll
    for (int j = 0; j < PER; j++) {
      const int gr = row0 + (tid >> 6) + 4 * j;
      v[j] = (src && gr < a.M) ? __ldg(src + (size_t)gr * ld) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < PER; j++)
      *reinterpret_cast<__nv_bfloat16*>(smem + OFF_A + sw128_offset((tid >> 6) + 4 * j, k, TILE_M)) = __float2bfloat16(v[j]);
  }
  fence_async_smem();
  __syncthreads();

  // Activation dumps for the backward pass, written from the shared-memory tile the epilogue just produced (while the next layer's MMAs
  // read the same tile): row-major [batch][256] with one full 512-byte row per warp instruction, and the [256][batch] copy as 16-byte
  // runs of eight consecutive batch rows per column (the accumulator fragments spread a row over four threads: their stores would be
  // 4-byte scatters for the transposed copy and quarter-used sectors for the row-major one).
  auto dump_tile = [&](__nv_bfloat16* d_rm, __nv_bfloat16* d_t, int ncols /*256: hidden activations (per net), 64: the input tile (shared by the nets)*/) {
    const int nrows = min(TILE_M, a.M - row0);
    const size_t nbase = ncols == HID ? (size_t)net : 0;
    if (d_rm) {
      if (lane * 8 < ncols)
        for (int r = warp; r < nrows; r += NTHR / 32) {
          const uint4 v = *reinterpret_cast<const uint4*>(smem + OFF_A + sw128_offset(r, lane * 8, TILE_M));
          *reinterpret_cast<uint4*>(d_rm + (nbase * a.M + row0 + r) * ncols + lane * 8) = v;
        }
    }
    if (d_t && tid < ncols) {
      const int c = tid;                                   // NTHR == HID: one column per thread
      __nv_bfloat16* dst = d_t + (nbase * ncols + c) * a.M + row0;
#pragma unroll 4
      for (int r0 = 0; r0 < TILE_M; r0 += 8) {
        uint32_t w[4];                                     // packed in registers (a local bf16[8] would live in local memory)
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const uint32_t lo = *reinterpret_cast<const uint16_t*>(smem + OFF_A + sw128_offset(r0 + 2 * i, c, TILE_M));
          const uint32_t hi = *reinterpret_cast<const uint16_t*>(smem + OFF_A + sw128_offset(r0 + 2 * i + 1, c, TILE_M));
          w[i] = lo | (hi << 16);
        }
        if (r0 + 8 <= nrows) *reinterpret_cast<uint4*>(dst + r0) = make_uint4(w[0], w[1], w[2], w[3]);
        else {
          uint16_t* d16 = reinterpret_cast<uint16_t*>(dst + r0);
#pragma unroll
          for (int i = 0; i < 8; i++) if (r0 + i < nrows) d16[i] = (uint16_t)(w[i >> 1] >> (16 * (i & 1)));
        }
      }
    }
  };
  // a layer over the K = 256 hidden width: 16 K-steps of 16, A = this warpgroup's 64 rows of the 4-panel tile, B = a [n_rows][256] operand image
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; i++) acc[i] = 0.f;
  auto mma_hidden_256 = [&](uint32_t sb) {
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 16; ks++)
      Wgmma<HID>::mma(acc, wg_desc(sAw + (ks >> 2) * (TILE_M * 128) + (ks & 3) * 32), wg_desc(sb + (ks >> 2) * (HID * 128) + (ks & 3) * 32), ks > 0);
    wg_commit();
  };
  auto mma_done = [&]() { wg_wait0(); wg_fence_acc(acc); };

  // ---- layer 1: [128 x 64] x [256 x 64]^T -> acc (each warpgroup its 64 rows)
  mbar_wait(bar_w1, 0);
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ks++) Wgmma<HID>::mma(acc, wg_desc(sAw + ks * 32), wg_desc(sW13 + ks * 32), ks > 0);
  wg_commit();
  if (a.save && net == 0 && (a.sv.x_rm || a.sv.x_t)) dump_tile(a.sv.x_rm, a.sv.x_t, 64);   // the input tile (panel 0), before epilogue 1 overwrites it
  mma_done();
  __syncthreads();   // both warpgroups are done with W1 and the input tile
  if (tid == 0) {    // W1 is consumed: reuse its region for W3
    mbar_expect_tx(bar_w3, SZ_W3 + (a.da ? SZ_W1A : 0u));
    bulk_g2s(sW13, img + IMG_W3, SZ_W3, bar_w3);
    if (a.da) bulk_g2s(sW13 + OFF_W1A_IN_W13, img + IMG_W1A, SZ_W1A, bar_w3);
  }
  // relu'(h1) of the thread's fragment (bit 4 j + 2 h + e of the 128: word j >> 3), kept for the input-gradient pass
  uint32_t m1[4] = {0u, 0u, 0u, 0u};
  // bias + ReLU in f32, bf16 back into the A-operand tile for the next layer (a warpgroup writes only the rows its own MMAs read)
  auto epilogue_hidden = [&](const float* b, bool keep_mask) {
#pragma unroll
    for (int j = 0; j < 32; j++) {
      const int c = 8 * j + fc0;
      const float b0 = b[c], b1 = b[c + 1];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const float v0 = fmaxf(acc[4 * j + 2 * h] + b0, 0.f), v1 = fmaxf(acc[4 * j + 2 * h + 1] + b1, 0.f);
        if (keep_mask) m1[j >> 3] |= ((v0 > 0.f ? 1u : 0u) | (v1 > 0.f ? 2u : 0u)) << (4 * (j & 7) + 2 * h);
        *reinterpret_cast<__nv_bfloat162*>(smem + OFF_A + sw128_offset(fr0 + 8 * h, c, TILE_M)) = __floats2bfloat162_rn(v0, v1);
      }
    }
  };
  epilogue_hidden(bias, a.da != nullptr);
  fence_async_smem();
  __syncthreads();

  // ---- layer 2: [128 x 256] x [256 x 256]^T -> acc
  mbar_wait(bar_w2, 0);
  mma_hidden_256(sW2);
  if (a.save) dump_tile(a.sv.h1_rm, a.sv.h1_t, HID);
  mma_done();
  __syncthreads();   // reads of W2 and of the h1 tile end before anything overwrites them
  if (a.da && tid == 0) {   // layer 2 has consumed W2: its region takes the W2^T image for the input-gradient pass
    mbar_expect_tx(bar_w2t, SZ_W2);
#pragma unroll
    for (int i = 0; i < 4; i++) bulk_g2s(sW2 + i * 32768u, img + IMG_W2T + (size_t)i * 32768u, 32768u, bar_w2t);
  }
  epilogue_hidden(bias + HID, false);
  fence_async_smem();
  __syncthreads();

  // ---- layer 3: [128 x 256] x [32 x 256]^T -> acc3
  float acc3[16];
#pragma unroll
  for (int i = 0; i < 16; i++) acc3[i] = 0.f;
  mbar_wait(bar_w3, 0);
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < 16; ks++)
    Wgmma<32>::mma(acc3, wg_desc(sAw + (ks >> 2) * (TILE_M * 128) + (ks & 3) * 32), wg_desc(sW13 + (ks >> 2) * (32 * 128) + (ks & 3) * 32), ks > 0);
  wg_commit();
  if (a.save) dump_tile(a.sv.h2_rm, a.sv.h2_t, HID);   // the head epilogue does not write the tile: no barrier needed
  wg_wait0();
  wg_fence_acc(acc3);
  {
    const float* b3 = bias + 2 * HID;
    const int od = a.out_dim;
    // RAW outputs (critics, BC, the actor's raw head) straight from the fragment
    if (a.raw || a.mode == B2Q_MLP_RAW) {
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int c = 8 * j + fc0 + e, gr = row0 + fr0 + 8 * h;
            if (c < od && gr < a.M) {
              const float y = acc3[4 * j + 2 * h + e] + b3[c];
              const size_t orow = (size_t)net * a.M + gr;
              if (a.raw) a.raw[orow * od + c] = y;
              if (a.mode == B2Q_MLP_RAW) a.out[orow * od + c] = y;
            }
          }
    }
    // PREDICT / SAMPLE (actor): the head needs a row's mean and log-std together, so the [128 x 32] result is staged row-wise in the W2
    // region (free: the input-gradient pass, the only later reader of that region, runs for RAW critics only).  BOTH threads of a row then
    // take every second action — the per-action tanh / exp / log / counter-RNG work is the longest stretch of the actor forward — and the
    // log-prob halves meet in shared memory.  All register indices are compile-time (no local arrays).
    if (a.mode != B2Q_MLP_RAW) {
      constexpr int LDS = 33;
      float* stage = reinterpret_cast<float*>(smem + OFF_W2);
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int e = 0; e < 2; e++) stage[(fr0 + 8 * h) * LDS + 8 * j + fc0 + e] = acc3[4 * j + 2 * h + e];
      __syncthreads();
      uint32_t r[32];
#pragma unroll
      for (int j = 0; j < 32; j++) r[j] = __float_as_uint(stage[trow * LDS + j]);
      float* slp = reinterpret_cast<float*>(smem + OFF_BAR + 64);            // [128] log-prob share of column half 1
      const size_t orow = (size_t)net * a.M + row;
      float lp = 0.f;
      if (row < a.M) {
        if ((od >> 1) == 12) lp = head_actions<12>(r, b3, a, row, orow, chalf);   // the A1's action dimension: every index compile-time
        else lp = head_actions<0>(r, b3, a, row, orow, chalf);
      }
      if (a.mode == B2Q_MLP_SAMPLE && a.logp) {
        if (chalf == 1) slp[trow] = lp;
        __syncthreads();
        if (chalf == 0 && row < a.M) a.logp[orow] = lp + slp[trow];
      }
    }
  }
  if (a.da) {
    // ---- input-gradient pass (out_dim == 1): unit output gradient back to the action columns of the input, on the same tile.
    __syncthreads();   // both warpgroups' layer-3 MMAs have read the h2 tile
    // (a) dh2 = W3 . relu'(h2), in place over the h2 tile.  Row 0 of the W3 operand image is W3 itself: 128 contiguous bytes per 64-column panel.
#pragma unroll 4
    for (int c0 = 128 * chalf; c0 < 128 * chalf + 128; c0 += 8) {
      uint8_t* hp = smem + OFF_A + sw128_offset(trow, c0, TILE_M);
      const uint4 hv = *reinterpret_cast<const uint4*>(hp);
      const uint4 wv = *reinterpret_cast<const uint4*>(smem + OFF_W13 + (c0 >> 6) * (32 * 128) + (c0 & 63) * 2);
      const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}, ww[4] = {wv.x, wv.y, wv.z, wv.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; j++) o[j] = ((hw[j] & 0x7fffu) ? (ww[j] & 0xffffu) : 0u) | ((hw[j] & 0x7fff0000u) ? (ww[j] & 0xffff0000u) : 0u);   // h2 = relu(.) >= 0: nonzero <=> positive
      *reinterpret_cast<uint4*>(hp) = make_uint4(o[0], o[1], o[2], o[3]);
    }
    fence_async_smem();
    __syncthreads();
    // (b) dh1 pre-mask = dh2 . W2  -> acc (B operand: the W2^T image)
    mbar_wait(bar_w2t, 0);
    mma_hidden_256(sW2);
    mma_done();
    // (c) dh1 = . relu'(h1) (bits kept from epilogue 1, same fragment positions) -> bf16 over this warpgroup's rows of the tile
#pragma unroll
    for (int j = 0; j < 32; j++) {
      const int c = 8 * j + fc0;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int bit = 4 * (j & 7) + 2 * h;
        const float v0 = ((m1[j >> 3] >> bit) & 1u) ? acc[4 * j + 2 * h] : 0.f, v1 = ((m1[j >> 3] >> (bit + 1)) & 1u) ? acc[4 * j + 2 * h + 1] : 0.f;
        *reinterpret_cast<__nv_bfloat162*>(smem + OFF_A + sw128_offset(fr0 + 8 * h, c, TILE_M)) = __floats2bfloat162_rn(v0, v1);
      }
    }
    fence_async_smem();
    __syncthreads();
    // (d) da = dh1 . W1[:, action]  -> accd (B operand: the W1A image, N = 16)
    float accd[8];
#pragma unroll
    for (int i = 0; i < 8; i++) accd[i] = 0.f;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 16; ks++)
      Wgmma<16>::mma(accd, wg_desc(sAw + (ks >> 2) * (TILE_M * 128) + (ks & 3) * 32), wg_desc(sW13 + OFF_W1A_IN_W13 + (ks >> 2) * (16 * 128) + (ks & 3) * 32), ks > 0);
    wg_commit();
    wg_wait0();
    wg_fence_acc(accd);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int gr = row0 + fr0 + 8 * h;
      if (gr < a.M) {
        float* dst = a.da + ((size_t)net * a.M + gr) * 16;
#pragma unroll
        for (int j = 0; j < 2; j++) *reinterpret_cast<float2*>(dst + 8 * j + fc0) = make_float2(accd[4 * j + 2 * h], accd[4 * j + 2 * h + 1]);
      }
    }
  }
}

// f32 nn.Linear weights -> one net's image: a thread per parameter, in the flat order the packer indexes
__global__ void b2q_mlp_pack_kernel(PackDst d, const float* w1, const float* b1, const float* w2, const float* b2, const float* w3, const float* b3) { pdl_sync();
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n) return;
  const float v = i < d.ob1 ? w1[i] : i < d.oW2 ? b1[i - d.ob1] : i < d.ob2 ? w2[i - d.oW2] : i < d.oW3 ? b2[i - d.ob2] : i < d.ob3 ? w3[i - d.oW3] : b3[i - d.ob3];
  pack_param(d, i, v);
}

}  // namespace

struct B2QMlp {
  int device, in_dim, out_dim, nets;
  int a_off = 0, a_dim = 0;
  uint8_t* img = nullptr;
  std::string err;
  int64_t launches = 0;
};

extern "C" {

int b2q_mlp_create(int device, int in_dim, int out_dim, int nets, B2QMlpHandle* out) {
  if (!out || in_dim < 1 || in_dim > B2Q_MLP_MAX_IN || out_dim < 1 || out_dim > B2Q_MLP_MAX_OUT || nets < 1 || nets > 8) return -1;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return -2;
  B2QMlp* h = new (std::nothrow) B2QMlp();
  if (!h) return -3;
  h->device = device; h->in_dim = in_dim; h->out_dim = out_dim; h->nets = nets;
  cudaSetDevice(device);
  if (cudaMalloc(&h->img, IMG_BYTES * nets) != cudaSuccess) { delete h; return -3; }
  cudaMemset(h->img, 0, IMG_BYTES * nets);
  if (cudaFuncSetAttribute(b2q_mlp_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES) != cudaSuccess) { cudaFree(h->img); delete h; return -2; }
  *out = h;
  return 0;
}
int b2q_mlp_destroy(B2QMlpHandle h) {
  if (!h) return -1;
  cudaSetDevice(h->device);
  cudaFree(h->img);
  delete h;
  return 0;
}
const char* b2q_mlp_last_error(B2QMlpHandle h) { return h ? h->err.c_str() : "null handle / create failed"; }
int64_t b2q_mlp_launch_count(B2QMlpHandle h) { return h ? h->launches : 0; }
int b2q_mlp_set_action_slice(B2QMlpHandle h, int a_off, int a_dim) {
  if (!h || a_off < 0 || a_dim < 0 || a_dim > 16 || a_off + a_dim > h->in_dim) return -1;
  h->a_off = a_off; h->a_dim = a_dim;
  return 0;
}
uint8_t* b2q_mlp_image(B2QMlpHandle h, int net) { return (h && net >= 0 && net < h->nets) ? h->img + (size_t)net * IMG_BYTES : nullptr; }

int b2q_mlp_set_weights(B2QMlpHandle h, int net, const float* w1, const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, void* stream) {
  if (!h || net < 0 || net >= h->nets || !w1 || !b1 || !w2 || !b2 || !w3 || !b3) { if (h) h->err = "b2q_mlp_set_weights: bad argument"; return -1; }
  const PackDst d = pack_dst(h->img + (size_t)net * IMG_BYTES, h->in_dim, h->out_dim, h->a_off, h->a_dim);
  pdl_launch(b2q_mlp_pack_kernel, dim3((d.n + 255) / 256), dim3(256), 0, (cudaStream_t)stream, d, w1, b1, w2, b2, w3, b3);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return -2; }
  return 0;
}

int b2q_mlp_forward_ex(B2QMlpHandle h, const float* in1, int in1_dim, const float* in2, int M, int mode, uint64_t seed, const float* eps, float* out,
                       float* logp, float* raw, const B2QMlpSaves* saves, float* da, const int* seed_ctr, void* stream) {
  if (!h || !in1 || !out || M < 1 || in1_dim < 1 || in1_dim > h->in_dim || (in1_dim < h->in_dim && !in2) || mode < 0 || mode > 2 ||
      (mode != B2Q_MLP_RAW && (h->out_dim & 1)) || (da && (h->out_dim != 1 || h->a_dim < 1 || saves))) { if (h) h->err = "b2q_mlp_forward: bad argument"; return -1; }
  { int cur = -1; if (cudaGetDevice(&cur) != cudaSuccess || cur != h->device) cudaSetDevice(h->device); }   // handles are per GPU
  FwdArgs a{in1, in2, in1_dim, h->in_dim, h->out_dim, M, mode, seed, eps, out, logp, raw, h->img, IMG_BYTES, B2QMlpSaves{}, 0, da, seed_ctr};
  if (saves) { a.sv = *saves; a.save = 1; }
  dim3 grid((M + TILE_M - 1) / TILE_M, h->nets);
  pdl_launch(b2q_mlp_fwd_kernel, dim3(grid), dim3(NTHR), SMEM_BYTES, (cudaStream_t)stream, a);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return -2; }
  return 0;
}
int b2q_mlp_forward(B2QMlpHandle h, const float* in1, int in1_dim, const float* in2, int M, int mode, uint64_t seed, const float* eps, float* out,
                    float* logp, float* raw, void* stream) {
  return b2q_mlp_forward_ex(h, in1, in1_dim, in2, M, mode, seed, eps, out, logp, raw, nullptr, nullptr, nullptr, stream);
}

}  // extern "C"
