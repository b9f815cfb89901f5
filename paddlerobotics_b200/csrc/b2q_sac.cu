// b2q_sac.cu — K5/K6: SAC update on the GPU (include/b2q_sac.h): critic + actor forward (fused wgmma MLP kernel of
// b2q_mlp.cu with activation dumps), backward GEMMs on wgmma tensor cores, fused elementwise epilogues, Adam and Polyak.
// Reference: SAC.learn / _critic_learn / _actor_learn / sync_target, ETGRL/alg/sac.py:77-118; torch.optim.Adam :55-58.
//
// Every backward product is phrased as C[MxN] (+)= A[MxK] . B[NxK]^T with both operands K-major bf16 (the layout the
// wgmma descriptors of b2q_tc.cuh address): weight gradients contract over the batch (K = batch, split-K across CTAs,
// f32 atomics), data gradients contract over the hidden width.  Activations are therefore kept in two bf16 layouts
// ([batch x width] and [width x batch]) written by the forward kernel's epilogue, and each weight matrix has a transposed
// bf16 copy refreshed by the optimiser kernel.
#include <cuda.h>
#include <cuda_runtime.h>
#include <map>
#include <tuple>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstring>
#include <new>
#include <string>
#include <vector>
#include "../../include/b2q_sac.h"
#include "b2q_mlp_internal.h"
#include "b2q_philox.cuh"
#include "b2q_tc.cuh"
#include "b2q_snapshot.h"

using namespace b2q_tc;
typedef __nv_bfloat16 bf16;

namespace {

constexpr int H = 256;

// ---------------------------------------------------------------------------------------------------------------------
// generic tensor-core GEMM  C[M x N] (+)= A[M x K] . B[N x K]^T   (bf16 K-major operands, f32 result), N tiled by BN <= 64
//
// Hopper feed: both operands arrive through TMA tensor maps (cp.async.bulk.tensor.2d, SWIZZLE_128B boxes of 64 K-elements: exactly
// the K-major shared-memory image the wgmma descriptors address; out-of-range rows / K are zero-filled by the TMA unit) into a 4-stage
// mbarrier ring that thread 0 keeps G_NSTAGE - 1 chunks ahead of the MMAs.  One warpgroup (128 threads) issues the wgmmas for the two
// 64-row halves of the 128-row tile (accumulators in registers), then the epilogue goes registers -> shared memory -> fully coalesced
// stores (or coalesced f32 reductions for the split-K weight gradients).
struct GemmArgs {
  float* C; int ldc;
  int M, N, K, BN, chunks_per_split, atomic;
  // ReLU-backward epilogue (mask_h != null; BN = 64, full 128-row tiles): instead of the f32 tile, write  dh = C . [h > 0]  as bf16 — row-major
  // [M][N] (dh_rm) and / or [N][M] (dh_t), either may be null — and add its column sums to db: the product never makes the f32 round trip
  // through HBM and the separate mask kernel drops out of the dependency chain
  const bf16* mask_h; bf16 *dh_rm, *dh_t; float* db;
};
constexpr int G_NSTAGE = 4;
constexpr uint32_t G_STAGE_A = 128 * 128, G_STAGE_B = 64 * 128, G_STAGE = G_STAGE_A + G_STAGE_B;   // bytes: 128 x 64 bf16 and BN(<=64) x 64 bf16
constexpr uint32_t G_SMEM = G_NSTAGE * G_STAGE + 128 + 1024;                                       // + barriers + alignment slack
constexpr int B2Q_GEMM_SPLIT_DIV = 8;                                                               // K chunks (of 64) per split-K CTA

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(bar) : "memory");
}

// WN: the MMA width (32 or 64) covering the tile's BN columns; B rows beyond BN only feed accumulator columns that are never stored
template <int WN>
__global__ void __launch_bounds__(128) b2q_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmArgs g) { pdl_sync();
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;                 // SWIZZLE_128B operand tiles want 1024-byte alignment
  uint8_t* smem = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t bar_full = sbase + G_NSTAGE * G_STAGE;
  const int row0 = blockIdx.x * 128, n0 = blockIdx.y * g.BN;   // output tile: 128 rows x BN columns
  const int nk_total = (g.K + 63) / 64;
  const int kc0 = blockIdx.z * g.chunks_per_split, kc1 = min(nk_total, kc0 + g.chunks_per_split), nk = kc1 - kc0;
  const uint32_t bytes = G_STAGE_A + (uint32_t)g.BN * 128u;
  auto load = [&](int kc) {   // thread 0: chunk kc of this split into its stage
    const int st = kc % G_NSTAGE;
    mbar_expect_tx(bar_full + 8 * st, bytes);
    tma_load_2d(sbase + st * G_STAGE, &tmA, (kc0 + kc) * 64, row0, bar_full + 8 * st);
    tma_load_2d(sbase + st * G_STAGE + G_STAGE_A, &tmB, (kc0 + kc) * 64, n0, bar_full + 8 * st);
  };
  if (tid == 0) {
    for (int i = 0; i < G_NSTAGE; i++) mbar_init(bar_full + 8 * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int kc = 0; kc < min(nk, G_NSTAGE); kc++) load(kc);
  }
  __syncthreads();
  if (nk <= 0) return;
  // accumulator fragments of the two 64-row halves (b2q_tc.cuh: d[4 j + 2 h + e] = row 16 warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e)
  float acc[2][WN / 2];
#pragma unroll
  for (int m = 0; m < 2; m++)
#pragma unroll
    for (int i = 0; i < WN / 2; i++) acc[m][i] = 0.f;
  for (int kc = 0; kc < nk; kc++) {
    const int st = kc % G_NSTAGE;
    mbar_wait(bar_full + 8 * st, (uint32_t)((kc / G_NSTAGE) & 1));
    const uint32_t sa = sbase + st * G_STAGE, sb = sa + G_STAGE_A;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ks++)
#pragma unroll
      for (int m = 0; m < 2; m++) Wgmma<WN>::mma(acc[m], wg_desc(sa + m * 64 * 128 + ks * 32), wg_desc(sb + ks * 32), (kc > 0 || ks > 0) ? 1u : 0u);
    wg_commit();
    wg_wait0();
    wg_fence_acc(acc[0]); wg_fence_acc(acc[1]);
    if (kc + G_NSTAGE < nk) {
      __syncthreads();                                   // every warp's MMAs have read the stage before it is refilled
      if (tid == 0) load(kc + G_NSTAGE);
    }
  }
  __syncthreads();                                       // the operand ring is drained: the epilogue reuses it as its staging tile
  const int fr = 16 * warp + (lane >> 2), fc = 2 * (lane & 3);
  if (g.mask_h) {
    constexpr int LDR = 72, LDT = 136;                                  // bf16 elements per staged row: 16-byte aligned
    bf16* t_rm = reinterpret_cast<bf16*>(smem);                          // [128][LDR]  rows x this CTA's 64 columns
    bf16* t_t = reinterpret_cast<bf16*>(smem + 128 * LDR * 2);           // [64][LDT]   columns x 128 rows
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r_ = 64 * m + fr + 8 * h;
        const bf16* hrow = g.mask_h + (size_t)(row0 + r_) * g.N + n0;
#pragma unroll
        for (int j = 0; j < WN / 8; j++) {
          const int c_ = 8 * j + fc;
          const __nv_bfloat162 hv = *reinterpret_cast<const __nv_bfloat162*>(hrow + c_);
          const bf16 o0 = __float2bfloat16(__bfloat162float(hv.x) > 0.f ? acc[m][4 * j + 2 * h] : 0.f);
          const bf16 o1 = __float2bfloat16(__bfloat162float(hv.y) > 0.f ? acc[m][4 * j + 2 * h + 1] : 0.f);
          __nv_bfloat162 o; o.x = o0; o.y = o1;
          *reinterpret_cast<__nv_bfloat162*>(t_rm + r_ * LDR + c_) = o;
          t_t[c_ * LDT + r_] = o0; t_t[(c_ + 1) * LDT + r_] = o1;
        }
      }
    __syncthreads();
    if (g.dh_rm)
      for (int i = tid; i < 128 * 8; i += 128) { const int r_ = i >> 3, sg = i & 7;
        *reinterpret_cast<uint4*>(g.dh_rm + (size_t)(row0 + r_) * g.N + n0 + sg * 8) = *reinterpret_cast<const uint4*>(t_rm + r_ * LDR + sg * 8); }
    if (g.dh_t)
      for (int i = tid; i < 64 * 16; i += 128) { const int c_ = i >> 4, sg = i & 15;
        *reinterpret_cast<uint4*>(g.dh_t + (size_t)(n0 + c_) * g.M + row0 + sg * 8) = *reinterpret_cast<const uint4*>(t_t + c_ * LDT + sg * 8); }
    if (g.db) {                                                          // column sums of the rounded values (what the weight-gradient GEMMs see)
      const int c_ = tid >> 1, hf = tid & 1;
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const uint4 v = *reinterpret_cast<const uint4*>(t_t + c_ * LDT + hf * 64 + k * 8);
        const bf16* vb = reinterpret_cast<const bf16*>(&v);
#pragma unroll
        for (int j = 0; j < 8; j++) sum += __bfloat162float(vb[j]);
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      if (hf == 0) atomicAdd(g.db + n0 + c_, sum);
    }
  } else {
    float* stile = reinterpret_cast<float*>(smem);                      // [128][BN + 1] floats
    const int ldt = g.BN + 1;
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int j = 0; j < WN / 8; j++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int c_ = 8 * j + fc + e;
            if (c_ < g.BN) stile[(64 * m + fr + 8 * h) * ldt + c_] = acc[m][4 * j + 2 * h + e];
          }
    __syncthreads();
    const int ncol = min(g.BN, g.N - n0), nrow = min(128, g.M - row0);
    for (int i = tid; i < nrow * ncol; i += 128) {
      const int r_ = i / ncol, c_ = i - r_ * ncol;
      float* c = g.C + (size_t)(row0 + r_) * g.ldc + n0 + c_;
      const float v = stile[r_ * ldt + c_];
      if (g.atomic) atomicAdd(c, v); else *c = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// elementwise / reduction kernels
// Vectorised tile kernels: a block walks SUBT sub-tiles of 32 batch rows x 256 hidden columns (256 threads: a warp handles one row at a
// time, each lane 8 consecutive columns — 16-byte bf16 / 2 x 16-byte f32 accesses, fully coalesced).  Column sums and the head's weight
// gradient are accumulated in registers / shared memory over the block's SUBT x 32 rows and flushed with ONE atomic per column per block
// (128 blocks at batch 8192: half the atomics and per-address contention of one block per 32 rows, and still one block per SM); the [width x batch]
// copy goes through the shared-memory tile as 64-byte row segments.
constexpr int SUBT = 2;
__device__ __forceinline__ void tile_transpose_out(bf16 (*tile)[H + 8], bf16* __restrict__ dh_t, int B, int b0, int nr) {
  __syncthreads();
  for (int i = threadIdx.x; i < H * 32; i += 256) { int c = i >> 5, r = i & 31; if (r < nr) dh_t[(size_t)c * B + b0 + r] = tile[r][c]; }
  __syncthreads();
}
__device__ __forceinline__ void colsum_flush(float (*csum)[H], const float* cs /*8 column sums of this thread*/, int chunk, int warp, float* db) {
#pragma unroll
  for (int j = 0; j < 8; j++) csum[warp][chunk * 8 + j] = cs[j];
  __syncthreads();
  if (db) { float t = 0.f; for (int w = 0; w < 8; w++) t += csum[w][threadIdx.x]; atomicAdd(db + threadIdx.x, t); }
  __syncthreads();
}
// critic head backward (out_dim = 1), same tiling: dh2[b,:] = dq[b] W3 masked by h2 > 0; dW3 += sum_b dq[b] h2[b,:]; db3 += sum_b dq; db2 += sum_b dh2
// A row's dq = 2 (q - tq)/B is computed in place (mse_loss mean reduction, loss += (q - tq)^2 / B), so no dq kernel sits on the dependency chain:
//   DQ_CRITIC: tq = r + gamma * term * (min(q1', q2') - alpha * logp')  (sac.py:85-95)
//   DQ_TWIN:   tq = qn[net][b], the expert's twin Q (BC.py:63-67)
enum { DQ_CRITIC = 0, DQ_TWIN = 1 };
struct DqSrc { int mode, net; const float *q /*[2][B]*/, *rew, *term, *qn /*[2][B]*/, *logpn; float gamma, alpha; float* loss; };
__device__ __forceinline__ float dq_of_row(const DqSrc& d, int b, int B, float& loss_acc) {
  const float tq = d.mode == DQ_TWIN ? d.qn[d.net * B + b] : d.rew[b] + d.gamma * d.term[b] * (fminf(d.qn[b], d.qn[B + b]) - d.alpha * d.logpn[b]);
  const float e = d.q[d.net * B + b] - tq;
  loss_acc += e * e / (float)B;
  return 2.f * e / (float)B;
}
__global__ void __launch_bounds__(256) k_head_bwd1(DqSrc src, const float* __restrict__ W3 /*[256]*/, const bf16* __restrict__ h2,
                                                   bf16* __restrict__ dh_rm, bf16* __restrict__ dh_t, float* dW3 /*[256]*/, float* db3 /*[1] or null*/, float* db2 /*[256] or null*/, int B) { pdl_sync();
  __shared__ __align__(16) bf16 tile[32][H + 8];
  __shared__ float csum[8][H];
  const int chunk = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float cs[8] = {0, 0, 0, 0, 0, 0, 0, 0}, acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, w[8];
#pragma unroll
  for (int j = 0; j < 8; j++) w[j] = W3[chunk * 8 + j];   // scalar loads: the second critic's parameter block starts at an odd float offset
  float sdq = 0.f, sloss = 0.f;
  for (int sub = 0; sub < SUBT; sub++) {
    const int b0 = (blockIdx.x * SUBT + sub) * 32, nr = min(32, B - b0);
    if (nr <= 0) break;
    uint4 hv[4]; float d[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int r = warp + 8 * k;
      if (r < nr) { hv[k] = *reinterpret_cast<const uint4*>(h2 + (size_t)(b0 + r) * H + chunk * 8); d[k] = dq_of_row(src, b0 + r, B, sloss); } else d[k] = 0.f;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int r = warp + 8 * k;
      if (r < nr) {
        const bf16* hb = reinterpret_cast<const bf16*>(&hv[k]);
        __align__(16) bf16 o[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float hf = __bfloat162float(hb[j]);
          acc[j] += d[k] * hf;
          o[j] = __float2bfloat16(hf > 0.f ? d[k] * w[j] : 0.f);
          cs[j] += __bfloat162float(o[j]);
        }
        *reinterpret_cast<uint4*>(dh_rm + (size_t)(b0 + r) * H + chunk * 8) = *reinterpret_cast<const uint4*>(o);
        *reinterpret_cast<uint4*>(&tile[r][chunk * 8]) = *reinterpret_cast<const uint4*>(o);
        sdq += d[k];
      }
    }
    tile_transpose_out(tile, dh_t, B, b0, nr);
  }
  colsum_flush(csum, acc, chunk, warp, dW3);                 // dW3: per-thread partials reduced over the 8 warps, one atomic per column
  if (db3 && chunk == 0) atomicAdd(db3, sdq);               // every lane of a warp holds the same rows: one lane per warp adds its dq sum
  if (chunk == 0) atomicAdd(src.loss, sloss);               // ... and its share of the critic loss
  colsum_flush(csum, cs, chunk, warp, db2);
}
// The head gradient dy = dloss/d[mean | raw_ls] leaves the dy kernels as bf16 in the two operand layouts the tensor-core GEMMs read
// (row-major [B][64] for dh2 = dy W3, [2A][B] for dW3 = dy^T h2); db3 = column sums of the rounded values.  A block = 32 batch rows x A
// action dimensions, one thread per element (coalesced f32 reads); the results meet in a shared-memory tile [2A][32] and leave as 64-byte
// runs per output row of the [2A][B] copy and contiguous 4A-byte rows of the row-major copy (no 2-byte scatters, no shared-memory atomics).
constexpr int DY_ROWS = 32;
__device__ __forceinline__ void dy_store_block(bf16 (*sT)[DY_ROWS], float l, int b0, int B, int A, bf16* dy_rm, bf16* dy_t, float* db3, float* loss) {
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  if ((threadIdx.x & 31) == 0 && l != 0.f) atomicAdd(loss, l);
  __syncthreads();
  const int t = threadIdx.x;
  if (t < 2 * A * 4) { const int row = t >> 2, seg = t & 3; *reinterpret_cast<uint4*>(dy_t + (size_t)row * B + b0 + seg * 8) = *reinterpret_cast<const uint4*>(&sT[row][seg * 8]); }
  for (int i = t; i < DY_ROWS * 2 * A; i += blockDim.x) { const int r = i / (2 * A), c = i - r * 2 * A; dy_rm[(size_t)(b0 + r) * 64 + c] = sT[c][r]; }
  if (db3 && t < 2 * A) {
    float sum = 0.f;
#pragma unroll
    for (int r = 0; r < DY_ROWS; r++) sum += __bfloat162float(sT[t][r]);
    atomicAdd(db3 + t, sum);
  }
}
// actor head: from raw y=[mean|raw_ls], eps, the critics' dQ_i/da (unit gradients) build dy and the loss   (B % 32 == 0; blockDim = 32 A)
__global__ void __launch_bounds__(384) k_actor_dy(const float* raw /*[B][2A]*/, const float* eps, const float* act /*[B][A] tanh(x)*/, const float* logp, const float* q /*[2][B]*/,
                           const float* da_c /*[B][16] (cols 0..A-1): dQ1/da*/, const float* da_c2 /*dQ2/da*/, float alpha,
                           bf16* dy_rm /*[B][64], cols >= 2A stay zero: A operand of the dh2 GEMM*/, bf16* dy_t /*[2A][B]: K-major A operand of the dW3 GEMM*/,
                           float* db3 /*[2A] += column sums of dy*/, float* loss, int B, int A, uint64_t seed, const int* seed_ctr /*eps == null: the forward's counter RNG draw*/) { pdl_sync();
  __shared__ __align__(16) bf16 sT[24][DY_ROWS];
  const int b0 = blockIdx.x * DY_ROWS, r = threadIdx.x / A, j = threadIdx.x - r * A, b = b0 + r, i = b * A + j;
  float l = 0.f;
  {
    const float q0 = q[b], q1 = q[B + b];
    if (j == 0) l = (alpha * logp[b] - fminf(q0, q1)) / (float)B;                  // sac.py:105-106
    const float a = act[i], rl = raw[(size_t)b * 2 * A + A + j];
    const float ls = fminf(fmaxf(rl, -20.f), 2.f), sd = expf(ls);
    const float e = eps ? eps[i] : b2q_philox::philox_normal(b2q_philox::effective_seed(seed, seed_ctr), (uint32_t)b, (uint32_t)j);
    const float dqa = (q0 <= q1 ? da_c : da_c2)[(size_t)b * 16 + j];              // d min(q1, q2)/da: torch.min routes to the first on ties (sac.py:104-106)
    const float ga = -dqa / (float)B + (alpha / (float)B) * (2.f * a / ((1.f - a * a) + 1e-6f));
    const float gx = ga * (1.f - a * a);
    const float gls = gx * sd * e - alpha / (float)B;
    const float gl = (rl > -20.f && rl < 2.f) ? gls : 0.f;                         // torch.clamp gradient
    sT[j][r] = __float2bfloat16(gx); sT[A + j][r] = __float2bfloat16(gl);
  }
  dy_store_block(sT, l, b0, B, A, dy_rm, dy_t, db3, loss);
}
// behaviour cloning head (alg/BC.py:53-59): loss = -mean_{b,j} log N(ref | mean, exp(ls)); dy = dloss/d[mean | raw_ls]
__global__ void __launch_bounds__(384) k_bc_dy(const float* raw /*[B][2A]*/, const float* ref /*[B][A]*/, bf16* dy_rm /*[B][64]*/, bf16* dy_t /*[2A][B]*/, float* db3, float* loss, int B, int A) { pdl_sync();
  __shared__ __align__(16) bf16 sT[24][DY_ROWS];
  const int b0 = blockIdx.x * DY_ROWS, r = threadIdx.x / A, j = threadIdx.x - r * A, b = b0 + r, i = b * A + j;
  const float inv = 1.f / (float)(B * A);
  const float mu = raw[(size_t)b * 2 * A + j], rl = raw[(size_t)b * 2 * A + A + j], ls = fminf(fmaxf(rl, -20.f), 2.f);
  const float d = ref[i] - mu, iv = expf(-2.f * ls);
  const float l = -(-0.5f * d * d * iv - ls - 0.9189385332046727f) * inv;
  const float g0 = -(d * iv) * inv, g1 = (rl > -20.f && rl < 2.f) ? -(d * d * iv - 1.f) * inv : 0.f;
  sT[j][r] = __float2bfloat16(g0); sT[A + j][r] = __float2bfloat16(g1);
  dy_store_block(sT, l, b0, B, A, dy_rm, dy_t, db3, loss);
}
// The optimiser kernels also REPACK what they update: each thread stores its new parameter through pack_param (b2q_mlp_internal.h) where the
// tensor-core kernels read it — the forward image of its net and the bf16 backward copies — so no pack kernel follows an optimiser step on the
// dependency chain.  k_pack does the same for parameters set from outside.
// Adam (torch.optim.Adam defaults: betas 0.9/0.999, eps 1e-8, no weight decay), sac.py:55-58, over the parameter blocks of one or two nets.
// The step counter lives on the device so that the whole learn() can be replayed from a CUDA graph.  `step` holds the number of COMPLETED
// optimiser steps: both Adam kernels of a learn use step + 1, and the one given `ticket` closes the step — its last block to finish advances
// the counter, so no increment kernel sits on the dependency chain and the kernel can run while another stream runs the Polyak update beside it.
__global__ void __launch_bounds__(256) k_adam_pack(float* p, const float* g, float* m, float* v, int n, float lr, float b1, float b2, float eps, int* step, int* ticket, PackDst2 dst) { pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float t = (float)(*step + 1), bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
    const float gi = g[i], mi = b1 * m[i] + (1.f - b1) * gi, vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float pn = p[i] - lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
    p[i] = pn;
    const unsigned per = dst.d[0].n, net = (unsigned)i / per;
    pack_param(dst.d[net], (unsigned)i - net * per, pn);
  }
  if (ticket) {
    __syncthreads();                                  // every thread of the block has read *step
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(ticket, 1) == (int)gridDim.x - 1) { *ticket = 0; *step += 1; }
    }
  }
}
__global__ void __launch_bounds__(256) k_polyak_pack(float* tgt, const float* src, int n, float tau, PackDst2 dst) { pdl_sync();   // sync_target, sac.py:112-118
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float tn = tau * src[i] + (1.f - tau) * tgt[i];
    tgt[i] = tn;
    const unsigned per = dst.d[0].n, net = (unsigned)i / per;
    pack_param(dst.d[net], (unsigned)i - net * per, tn);
  }
}
__global__ void __launch_bounds__(256) k_pack(const float* p, int n, PackDst2 dst) { pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const unsigned per = dst.d[0].n, net = (unsigned)i / per;
    pack_param(dst.d[net], (unsigned)i - net * per, p[i]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
struct Net {            // one 3-layer MLP: flat f32 params [W1|b1|W2|b2|W3|b3]
  int in_dim, od;
  size_t oW1, ob1, oW2, ob2, oW3, ob3, n;
  void layout(int in, int o) { in_dim = in; od = o; oW1 = 0; ob1 = oW1 + (size_t)H * in; oW2 = ob1 + H; ob2 = oW2 + (size_t)H * H; oW3 = ob2 + H; ob3 = oW3 + (size_t)o * H; n = ob3 + o; }
};

}  // namespace

struct B2QSac {
  int device, D, A, B;
  float gamma, tau, alpha, lr_a, lr_c;
  Net an, cn;
  // params: actor [an.n], critic [2][cn.n], target critic [2][cn.n]; grads, adam m/v
  float *p_actor = nullptr, *p_critic = nullptr, *p_target = nullptr, *g_actor = nullptr, *g_critic = nullptr, *m_a = nullptr, *v_a = nullptr, *m_c = nullptr, *v_c = nullptr;
  B2QMlpHandle mlp_actor = nullptr, mlp_critic = nullptr, mlp_target = nullptr;
  // bf16 backward weights per net (0 actor, 1 c1, 2 c2)
  bf16 *W2T[3] = {0, 0, 0}, *W3T[3] = {0, 0, 0}, *W1A[3] = {0, 0, 0};
  // activation dumps: critic (2 nets) and actor
  bf16 *xc_t = nullptr, *hc1_rm = nullptr, *hc1_t = nullptr, *hc2_rm = nullptr, *hc2_t = nullptr;
  bf16 *xa_t = nullptr, *ha1_rm = nullptr, *ha1_t = nullptr, *ha2_rm = nullptr, *ha2_t = nullptr;
  bf16 *dh_rm = nullptr, *dh_t = nullptr, *dy_bf = nullptr, *dy_rm = nullptr;
  bf16 *dh_rm2 = nullptr, *dh_t2 = nullptr;   // second scratch set: the twin critics' backward chains run on two streams
  cudaStream_t side = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaStream_t aux[2] = {nullptr, nullptr}; cudaEvent_t ev_aux[4] = {nullptr, nullptr, nullptr, nullptr};   // per-chain helper streams: dW2 GEMM beside the dh1 -> dW1 chain
  bf16 *dh1_rm[2] = {nullptr, nullptr}, *dh1_t[2] = {nullptr, nullptr};                                      // layer-1 gradients (separate from dh2 so both GEMM branches can run)
  float *q = nullptr, *qn = nullptr, *next_a = nullptr, *next_logp = nullptr, *cur_a = nullptr, *cur_logp = nullptr, *raw_a = nullptr,
        *da_c = nullptr, *losses = nullptr;
  std::vector<void*> allocs;
  void* tmap_cache = nullptr;   // TmapCache*: TMA tensor maps of the GEMM operands
  int* d_step = nullptr;
  int64_t launches = 0;
  bool actor_grad_dirty = false;   // g_actor holds a gradient that no phase 0 has cleared yet
  std::string err;
};

namespace {

template <typename T> bool dalloc(B2QSac* s, T** p, size_t count) {
  void* v = nullptr;
  if (cudaMalloc(&v, count * sizeof(T)) != cudaSuccess) return false;
  cudaMemset(v, 0, count * sizeof(T));
  s->allocs.push_back(v);
  *p = (T*)v;
  return true;
}

// Fork / join of an internal side stream off the caller's stream (plain events: also legal inside a stream capture, where
// they become graph edges).  The twin critics' chains are independent and each kernel is latency-bound on a few SMs, so
// running them side by side nearly halves that part of a learn step.
void fork(B2QSac* s, cudaStream_t st) { cudaEventRecord(s->ev_fork, st); cudaStreamWaitEvent(s->side, s->ev_fork, 0); }
void join(B2QSac* s, cudaStream_t st) { cudaEventRecord(s->ev_join, s->side); cudaStreamWaitEvent(st, s->ev_join, 0); }

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    return (EncodeTiledFn)p;
  }();
  return fn;
}
// 2-D bf16 tensor map of a row-major [rows][cols] matrix with leading dimension ld: box = 64 K-elements (128 bytes, the swizzle span) x box_rows
bool make_tmap(CUtensorMap* tm, const bf16* base, int rows, int cols, int ld, int box_rows) {
  EncodeTiledFn enc = encode_tiled();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ld * sizeof(bf16)};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows}, estr[2] = {1u, 1u};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
struct TmapCache { std::map<std::tuple<const void*, int, int, int, int>, CUtensorMap> m; };
TmapCache& tmaps(B2QSac* s) { if (!s->tmap_cache) s->tmap_cache = new TmapCache(); return *static_cast<TmapCache*>(s->tmap_cache); }

struct ReluEpi { const bf16* h; bf16 *dh_rm, *dh_t; float* db; };
int gemm(B2QSac* s, cudaStream_t st, const bf16* A, int lda, const bf16* Bm, int ldb, float* C, int ldc, int M, int N, int K, bool splitk, int a_rows = 0,
         const ReluEpi* epi = nullptr) {
  GemmArgs g; g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
  g.mask_h = nullptr; g.dh_rm = g.dh_t = nullptr; g.db = nullptr;
  if (epi) {
    if (splitk || (M % 128) || (N % 64)) { s->err = "relu epilogue needs full 128 x 64 tiles and no split-K"; return -2; }
    g.mask_h = epi->h; g.dh_rm = epi->dh_rm; g.dh_t = epi->dh_t; g.db = epi->db;
  }
  g.BN = ((N + 15) / 16) * 16;
  if (g.BN > 64) g.BN = 64;                              // N tiled by 64 (grid.y): more CTAs on these latency-bound shapes, 8 KB B panel per k-chunk
  const int ntiles = (N + g.BN - 1) / g.BN;
  int nk = (K + 63) / 64, splits = 1;
  if (splitk) { splits = nk / B2Q_GEMM_SPLIT_DIV; if (splits < 1) splits = 1; if (splits > 64) splits = 64; }
  g.chunks_per_split = (nk + splits - 1) / splits;
  splits = (nk + g.chunks_per_split - 1) / g.chunks_per_split;
  g.atomic = splits > 1 ? 1 : 0;
  // tensor maps are cached per (pointer, shape): the learner's buffers are fixed, so each map is encoded once
  auto get = [&](const bf16* p, int rows, int ld, int box_rows) -> const CUtensorMap* {
    auto key = std::make_tuple((const void*)p, rows, K, ld, box_rows);
    auto& mp = tmaps(s).m;
    auto it = mp.find(key);
    if (it == mp.end()) {
      CUtensorMap tm;
      if (!make_tmap(&tm, p, rows, K, ld, box_rows)) return nullptr;
      it = mp.emplace(key, tm).first;
    }
    return &it->second;
  };
  const CUtensorMap* ta = get(A, a_rows > M ? a_rows : M, lda, 128);   // a_rows: the operand buffer holds that many (zero) rows, so the 128-row box stays inside it
  const CUtensorMap* tb = get(Bm, N, ldb, g.BN);
  if (!ta || !tb) { s->err = "cuTensorMapEncodeTiled failed"; return -2; }
  // split-K products accumulate with f32 atomics: C must be zero on entry (every caller targets the gradient bucket, cleared once per learn)
  dim3 grid((M + 127) / 128, ntiles, splits);
  if (g.BN <= 32) pdl_launch(b2q_gemm_kernel<32>, dim3(grid), dim3(128), G_SMEM, st, *ta, *tb, g);
  else pdl_launch(b2q_gemm_kernel<64>, dim3(grid), dim3(128), G_SMEM, st, *ta, *tb, g);
  s->launches++;
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// Where the packer stores each net of a parameter group: the actor (one net; d[1] repeats d[0]), the critics, or the target critics
// (forward images only: nothing differentiates through them).
enum { NETS_ACTOR = 0, NETS_CRITIC = 1, NETS_TARGET = 2 };
PackDst2 dst_of(const B2QSac* s, int group) {
  const bool actor = group == NETS_ACTOR, crit = group == NETS_CRITIC;
  const Net& nt = actor ? s->an : s->cn;
  const B2QMlpHandle mlp = actor ? s->mlp_actor : crit ? s->mlp_critic : s->mlp_target;
  PackDst2 r;
  for (int i = 0; i < 2; i++) {
    PackDst& d = r.d[i];
    d = pack_dst(b2q_mlp_image(mlp, actor ? 0 : i), nt.in_dim, nt.od, crit ? s->D : 0, crit ? s->A : 0);
    if (group != NETS_TARGET) { const int bw = actor ? 0 : 1 + i; d.W2T = s->W2T[bw]; d.W3T = s->W3T[bw]; d.W1A = s->W1A[bw]; }
  }
  return r;
}

}  // namespace

namespace {
// one MLP's weight-gradient chain after its head backward: dW2 (split-K GEMM over the batch) runs on the helper stream `ax`
// beside  dh1 = (dh2 W2) . relu'  ->  dW1  on `st`
int hidden_backward(B2QSac* s, cudaStream_t st, int slot, const bf16* dh2_rm, const bf16* dh2_t, const bf16* h1_rm, const bf16* h1_t, const bf16* x_t,
                    const bf16* W2T, float* gW2, float* gb1, float* gW1, int in_dim) {
  const int B = s->B;
  cudaStream_t ax = s->aux[slot];
  cudaEventRecord(s->ev_aux[2 * slot], st); cudaStreamWaitEvent(ax, s->ev_aux[2 * slot], 0);
  if (gemm(s, ax, dh2_t, B, h1_t, B, gW2, H, H, H, B, true)) return -2;
  cudaEventRecord(s->ev_aux[2 * slot + 1], ax);
  const ReluEpi epi{h1_rm, nullptr, s->dh1_t[slot], gb1};                                   // dh1 = (dh2 W2) . relu' and db1 in the GEMM's epilogue; only dW1 reads it: [width][batch] copy
  if (gemm(s, st, dh2_rm, H, W2T, H, nullptr, H, B, H, H, false, 0, &epi)) return -2;
  if (gemm(s, st, s->dh1_t[slot], B, x_t, B, gW1, in_dim, H, in_dim, B, true)) return -2;
  cudaStreamWaitEvent(st, s->ev_aux[2 * slot + 1], 0);
  s->launches += 3;
  return 0;
}
// weight gradients of both critics from the dq of `src` and the activation dumps of the last critic forward
int critic_backward(B2QSac* s, cudaStream_t st0, DqSrc src) {
  const int B = s->B; const Net& cn = s->cn;
  fork(s, st0);
  for (int i = 0; i < 2; i++) {
    cudaStream_t st = i ? s->side : st0;
    bf16 *dh_rm = i ? s->dh_rm2 : s->dh_rm, *dh_t = i ? s->dh_t2 : s->dh_t;
    float* g = s->g_critic + (size_t)i * cn.n; const float* p = s->p_critic + (size_t)i * cn.n;
    const bf16 *h1 = s->hc1_rm + (size_t)i * B * H, *h1t = s->hc1_t + (size_t)i * B * H, *h2 = s->hc2_rm + (size_t)i * B * H;
    src.net = i;
    pdl_launch(k_head_bwd1, dim3((B + 32 * SUBT - 1) / (32 * SUBT)), dim3(H), 0, st, src, p + cn.oW3, h2, dh_rm, dh_t, g + cn.oW3, g + cn.ob3, g + cn.ob2, B);   // dh2, dW3, db3, db2
    s->launches++;
    if (hidden_backward(s, st, i, dh_rm, dh_t, h1, h1t, s->xc_t, s->W2T[1 + i], g + cn.oW2, g + cn.ob1, g + cn.oW1, cn.in_dim)) return -2;
  }
  join(s, st0);
  return 0;
}
// actor weight gradients from dy [B][2A] and the activation dumps of the last actor forward
int actor_backward(B2QSac* s, cudaStream_t st) {
  const int B = s->B, A = s->A; const Net& an = s->an;
  float* g = s->g_actor;
  // dW3 = dy^T . h2 (contracted over the batch) is a split-K tensor-core GEMM on the helper stream — A = dy^T as bf16 [2A (padded to 128)][B] written
  // by the dy kernel, B = the [width x batch] dump of h2 — beside the head backward, which keeps dh2, db3 and db2
  cudaEventRecord(s->ev_aux[2], st); cudaStreamWaitEvent(s->aux[1], s->ev_aux[2], 0);
  if (gemm(s, s->aux[1], s->dy_bf, B, s->ha2_t, B, g + an.oW3, H, 2 * A, H, B, true, 128)) return -2;
  cudaEventRecord(s->ev_aux[3], s->aux[1]);
  // dh2 = (dy W3) . relu'(h2), db2: a K = 64 tensor-core GEMM (A = dy row-major, zero-padded; B = W3^T [256][64]) with the masking epilogue
  const ReluEpi epi{s->ha2_rm, s->dh_rm, s->dh_t, g + an.ob2};
  if (gemm(s, st, s->dy_rm, 64, s->W3T[0], 64, nullptr, H, B, H, 64, false, 0, &epi)) return -2;
  const int rc = hidden_backward(s, st, 0, s->dh_rm, s->dh_t, s->ha1_rm, s->ha1_t, s->xa_t, s->W2T[0], g + an.oW2, g + an.ob1, g + an.oW1, an.in_dim);
  cudaStreamWaitEvent(st, s->ev_aux[3], 0);
  return rc;
}
// the bf16 tensor-core operand images of all three parameter groups from the f32 parameters (b2q_sac_set_params, b2q_sac_snapshot_load)
int repack_all(B2QSac* s, cudaStream_t st) {
  const int na = (int)s->an.n, nc = (int)(2 * s->cn.n);
  pdl_launch(k_pack, dim3((na + 255) / 256), dim3(256), 0, st, s->p_actor, na, dst_of(s, NETS_ACTOR));
  pdl_launch(k_pack, dim3((nc + 255) / 256), dim3(256), 0, st, s->p_critic, nc, dst_of(s, NETS_CRITIC));
  pdl_launch(k_pack, dim3((nc + 255) / 256), dim3(256), 0, st, s->p_target, nc, dst_of(s, NETS_TARGET));
  s->launches += 3;
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// ---- learner snapshot (b2q_sac_snapshot_*): header, then the float buffers of sac_parts() in order, then d_step [2] (padded to 16 bytes)
constexpr uint32_t SAC_SNAP_VERSION = 1;
struct SacSnapHeader {
  char magic[8];
  uint32_t version, header_bytes;
  int64_t total_bytes;
  int32_t obs_dim, act_dim, batch, pad_;
  float gamma, tau, alpha, actor_lr, critic_lr;
};
#define B2Q_SAC_FIELD(f, name) b2q_snap::Field{name, offsetof(SacSnapHeader, f), sizeof(((SacSnapHeader*)nullptr)->f)}
const b2q_snap::Field SAC_SNAP_FIELDS[] = {
    B2Q_SAC_FIELD(magic, "magic"), B2Q_SAC_FIELD(version, "version"), B2Q_SAC_FIELD(header_bytes, "header size"), B2Q_SAC_FIELD(total_bytes, "size"),
    B2Q_SAC_FIELD(obs_dim, "obs_dim"), B2Q_SAC_FIELD(act_dim, "act_dim"), B2Q_SAC_FIELD(batch, "batch"), B2Q_SAC_FIELD(gamma, "gamma"),
    B2Q_SAC_FIELD(tau, "tau"), B2Q_SAC_FIELD(alpha, "alpha"), B2Q_SAC_FIELD(actor_lr, "actor_lr"), B2Q_SAC_FIELD(critic_lr, "critic_lr"),
};
struct SacPart { float* p; size_t n; };
// actor, critic, target, Adam m/v of the actor and of the critic, the loss buffer
void sac_parts(const B2QSac* s, SacPart out[8]) {
  const size_t na = s->an.n, nc = 2 * s->cn.n;
  out[0] = {s->p_actor, na}; out[1] = {s->p_critic, nc}; out[2] = {s->p_target, nc}; out[3] = {s->m_a, na};
  out[4] = {s->v_a, na}; out[5] = {s->m_c, nc}; out[6] = {s->v_c, nc}; out[7] = {s->losses, 4};
}
size_t sac_payload_floats(const B2QSac* s) {   // the blob's size follows the part list that save and load walk
  SacPart parts[8]; sac_parts(s, parts);
  size_t n = 0;
  for (const SacPart& q : parts) n += q.n;
  return n;
}
int64_t sac_snapshot_bytes(const B2QSac* s) { return (int64_t)(b2q_snap::HDR_BYTES + sac_payload_floats(s) * sizeof(float) + 16); }
SacSnapHeader sac_header(const B2QSac* s) {
  SacSnapHeader h;
  std::memset(&h, 0, sizeof h);
  std::memcpy(h.magic, "B2QSAC\0\0", 8);
  h.version = SAC_SNAP_VERSION; h.header_bytes = (uint32_t)b2q_snap::HDR_BYTES; h.total_bytes = sac_snapshot_bytes(s);
  h.obs_dim = s->D; h.act_dim = s->A; h.batch = s->B; h.gamma = s->gamma; h.tau = s->tau; h.alpha = s->alpha; h.actor_lr = s->lr_a; h.critic_lr = s->lr_c;
  return h;
}

}  // namespace

extern "C" {

int b2q_sac_create(int device, int obs_dim, int act_dim, int batch, float gamma, float tau, float alpha, float actor_lr, float critic_lr, B2QSacHandle* out) {
  if (!out || obs_dim < 1 || act_dim < 1 || act_dim > 12 || obs_dim + act_dim > 64 || batch < 128 || batch % 128 != 0) return -1;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return -2;
  cudaSetDevice(device);
  B2QSac* s = new (std::nothrow) B2QSac();
  if (!s) return -3;
  s->device = device; s->D = obs_dim; s->A = act_dim; s->B = batch; s->gamma = gamma; s->tau = tau; s->alpha = alpha; s->lr_a = actor_lr; s->lr_c = critic_lr;
  s->an.layout(obs_dim, 2 * act_dim); s->cn.layout(obs_dim + act_dim, 1);
  const size_t Bz = batch;
  // ONE flat gradient bucket [actor | critic 1 | critic 2] (SURVEY §8e collective 2: a single ncclAllReduce over 248 602 floats at obs 49)
  bool ok = dalloc(s, &s->p_actor, s->an.n) && dalloc(s, &s->g_actor, s->an.n + 2 * s->cn.n) && dalloc(s, &s->m_a, s->an.n) && dalloc(s, &s->v_a, s->an.n) &&
            dalloc(s, &s->p_critic, 2 * s->cn.n) && dalloc(s, &s->p_target, 2 * s->cn.n) && dalloc(s, &s->m_c, 2 * s->cn.n) && dalloc(s, &s->v_c, 2 * s->cn.n);
  if (ok) s->g_critic = s->g_actor + s->an.n;
  for (int i = 0; i < 3 && ok; i++) ok = dalloc(s, &s->W2T[i], (size_t)H * H) && dalloc(s, &s->W3T[i], (size_t)H * 64) && dalloc(s, &s->W1A[i], (size_t)16 * H);
  ok = ok && dalloc(s, &s->xc_t, 64 * Bz) && dalloc(s, &s->hc1_rm, 2 * Bz * H) && dalloc(s, &s->hc1_t, 2 * Bz * H) && dalloc(s, &s->hc2_rm, 2 * Bz * H) &&
       dalloc(s, &s->hc2_t, 2 * Bz * H) && dalloc(s, &s->xa_t, 64 * Bz) && dalloc(s, &s->ha1_rm, Bz * H) && dalloc(s, &s->ha1_t, Bz * H) &&
       dalloc(s, &s->ha2_rm, Bz * H) && dalloc(s, &s->ha2_t, Bz * H) && dalloc(s, &s->dh_rm, Bz * H) && dalloc(s, &s->dh_t, Bz * H) && dalloc(s, &s->dy_bf, Bz * 128) && dalloc(s, &s->dy_rm, Bz * 64) &&
       dalloc(s, &s->q, 2 * Bz) && dalloc(s, &s->qn, 2 * Bz) && dalloc(s, &s->next_a, Bz * 12) &&
       dalloc(s, &s->next_logp, Bz) && dalloc(s, &s->cur_a, Bz * 12) && dalloc(s, &s->cur_logp, Bz) && dalloc(s, &s->raw_a, Bz * 24) && dalloc(s, &s->da_c, 2 * Bz * 16) &&
       dalloc(s, &s->losses, 4) && dalloc(s, &s->d_step, 2 /*step | block ticket of the closing Adam*/) &&
       dalloc(s, &s->dh_rm2, Bz * H) && dalloc(s, &s->dh_t2, Bz * H) &&
       dalloc(s, &s->dh1_rm[0], Bz * H) && dalloc(s, &s->dh1_t[0], Bz * H) && dalloc(s, &s->dh1_rm[1], Bz * H) && dalloc(s, &s->dh1_t[1], Bz * H);
  for (int i = 0; i < 2 && ok; i++) ok = cudaStreamCreateWithFlags(&s->aux[i], cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; i < 4 && ok; i++) ok = cudaEventCreateWithFlags(&s->ev_aux[i], cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&s->side, cudaStreamNonBlocking) == cudaSuccess && cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming) == cudaSuccess &&
       cudaEventCreateWithFlags(&s->ev_join, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && b2q_mlp_create(device, obs_dim, 2 * act_dim, 1, &s->mlp_actor) == 0 && b2q_mlp_create(device, obs_dim + act_dim, 1, 2, &s->mlp_critic) == 0 &&
       b2q_mlp_create(device, obs_dim + act_dim, 1, 2, &s->mlp_target) == 0 &&
       b2q_mlp_set_action_slice(s->mlp_critic, obs_dim, act_dim) == 0;
  ok = ok && cudaFuncSetAttribute(b2q_gemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM) == cudaSuccess &&
       cudaFuncSetAttribute(b2q_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM) == cudaSuccess;
  if (!ok) { b2q_sac_destroy(s); return -3; }
  *out = s;
  return 0;
}

int b2q_sac_destroy(B2QSacHandle s) {
  if (!s) return -1;
  cudaSetDevice(s->device);
  for (void* p : s->allocs) cudaFree(p);
  if (s->side) cudaStreamDestroy(s->side);
  for (int i = 0; i < 2; i++) if (s->aux[i]) cudaStreamDestroy(s->aux[i]);
  for (int i = 0; i < 4; i++) if (s->ev_aux[i]) cudaEventDestroy(s->ev_aux[i]);
  if (s->ev_fork) cudaEventDestroy(s->ev_fork);
  if (s->ev_join) cudaEventDestroy(s->ev_join);
  if (s->mlp_actor) b2q_mlp_destroy(s->mlp_actor);
  if (s->mlp_critic) b2q_mlp_destroy(s->mlp_critic);
  if (s->mlp_target) b2q_mlp_destroy(s->mlp_target);
  delete static_cast<TmapCache*>(s->tmap_cache);
  delete s;
  return 0;
}
const char* b2q_sac_last_error(B2QSacHandle s) { return s ? s->err.c_str() : "null handle"; }
int64_t b2q_sac_launch_count(B2QSacHandle s) { return s ? s->launches : 0; }
int b2q_sac_param_count(B2QSacHandle s, int which) { return !s ? -1 : (which == 0 ? (int)s->an.n : (int)(2 * s->cn.n)); }

int b2q_sac_set_params(B2QSacHandle s, const float* actor, const float* critic, const float* target, void* stream) {
  if (!s) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (actor) cudaMemcpyAsync(s->p_actor, actor, s->an.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (critic) cudaMemcpyAsync(s->p_critic, critic, 2 * s->cn.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (target) cudaMemcpyAsync(s->p_target, target, 2 * s->cn.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  else if (critic) cudaMemcpyAsync(s->p_target, critic, 2 * s->cn.n * sizeof(float), cudaMemcpyDeviceToDevice, st);   // MujocoAgent: sync_target(decay=0)
  return repack_all(s, st);
}
int b2q_sac_get_params(B2QSacHandle s, float* actor, float* critic, float* target, void* stream) {
  if (!s) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (actor) cudaMemcpyAsync(actor, s->p_actor, s->an.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (critic) cudaMemcpyAsync(critic, s->p_critic, 2 * s->cn.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (target) cudaMemcpyAsync(target, s->p_target, 2 * s->cn.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  return 0;
}
int b2q_sac_get_grads(B2QSacHandle s, float* actor, float* critic, void* stream) {
  if (!s) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (actor) cudaMemcpyAsync(actor, s->g_actor, s->an.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (critic) cudaMemcpyAsync(critic, s->g_critic, 2 * s->cn.n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  return 0;
}

// phase 0: critic gradients (g_critic, losses[0]); phase 1: Adam on the critic; phase 2: actor gradients (g_actor, losses[1]);
// phase 3: Adam on the actor + Polyak.  b2q_sac_learn runs 0..3; the data-parallel learner all-reduces g_* between phases.
int b2q_sac_phase(B2QSacHandle s, int phase, const float* obs, const float* act, const float* rew, const float* next_obs, const float* term,
                  const float* eps_next, const float* eps_cur, uint64_t seed, void* stream) {
  if (!s) return -1;
  if (phase < 0 || phase > 3) return -1;
  if (phase == 2 && !obs) return -1;
  cudaSetDevice(s->device);                          // handles are per GPU
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s->B, A = s->A, D = s->D;
  const Net& an = s->an; const Net& cn = s->cn;
  if (phase == 0) {
    if (!obs || !act || !rew || !next_obs || !term) return -1;
    // target: next action ~ pi(next_obs), twin target Q (sac.py:85-91)
    fork(s, st);
    // ONE clear of the whole flat bucket [actor | critics] and the loss accumulators, after the fork: the caller's stream has slack here (the
    // side stream carries the longer chain), and phase 2 then starts without a memset node between the critics' Adam and the actor forward
    cudaMemsetAsync(s->losses, 0, 4 * sizeof(float), st);
    cudaMemsetAsync(s->g_actor, 0, (an.n + 2 * cn.n) * sizeof(float), st);
    s->actor_grad_dirty = false;
    if (b2q_mlp_forward_ex(s->mlp_actor, next_obs, D, nullptr, B, B2Q_MLP_SAMPLE, seed * 2 + 1, eps_next, s->next_a, s->next_logp, nullptr, nullptr, nullptr, s->d_step, s->side)) return -2;
    if (b2q_mlp_forward(s->mlp_target, next_obs, D, s->next_a, B, B2Q_MLP_RAW, 0, nullptr, s->qn, nullptr, nullptr, s->side)) return -2;
    // current Q with activation dumps (independent of the target chain: main stream)
    B2QMlpSaves sv = {nullptr /*x row-major: no consumer*/, s->xc_t, s->hc1_rm, s->hc1_t, s->hc2_rm, s->hc2_t};
    if (b2q_mlp_forward_ex(s->mlp_critic, obs, D, act, B, B2Q_MLP_RAW, 0, nullptr, s->q, nullptr, nullptr, &sv, nullptr, nullptr, st)) return -2;
    join(s, st);
    s->launches += 3;
    DqSrc src{DQ_CRITIC, 0, s->q, rew, term, s->qn, s->next_logp, s->gamma, s->alpha, s->losses + 0};   // target Q and dq are computed inside the head backward
    if (critic_backward(s, st, src)) return -2;
  } else if (phase == 1 || phase == 3) {
    const float b1 = 0.9f, b2 = 0.999f;
    if (phase == 1) {                                 // critics: Adam + repack (forward images and backward copies) in one kernel
      int n = (int)(2 * cn.n);
      pdl_launch(k_adam_pack, dim3((n + 255) / 256), dim3(256), 0, st, s->p_critic, s->g_critic, s->m_c, s->v_c, n, s->lr_c, b1, b2, 1e-8f, s->d_step, (int*)nullptr, dst_of(s, NETS_CRITIC));
      s->launches++;
    } else {                                          // actor Adam + repack on the caller's stream, Polyak + repack of the targets beside it
      int n = (int)an.n, nc = (int)(2 * cn.n);
      fork(s, st);
      pdl_launch(k_polyak_pack, dim3((nc + 255) / 256), dim3(256), 0, s->side, s->p_target, s->p_critic, nc, s->tau, dst_of(s, NETS_TARGET));
      pdl_launch(k_adam_pack, dim3((n + 255) / 256), dim3(256), 0, st, s->p_actor, s->g_actor, s->m_a, s->v_a, n, s->lr_a, b1, b2, 1e-8f, s->d_step, s->d_step + 1, dst_of(s, NETS_ACTOR));
      join(s, st);
      s->launches += 2;
    }
  } else if (phase == 2) {
    if (!obs) return -1;
    if (s->actor_grad_dirty) cudaMemsetAsync(s->g_actor, 0, an.n * sizeof(float), st);   // only when no phase 0 cleared the bucket since the last actor gradient
    s->actor_grad_dirty = true;
    // a ~ pi(obs) with dumps; Q(obs, a) with dumps (sac.py:102-106)
    B2QMlpSaves sa = {nullptr /*x row-major: no consumer*/, s->xa_t, s->ha1_rm, s->ha1_t, s->ha2_rm, s->ha2_t};
    if (b2q_mlp_forward_ex(s->mlp_actor, obs, D, nullptr, B, B2Q_MLP_SAMPLE, seed * 2, eps_cur, s->cur_a, s->cur_logp, s->raw_a, &sa, nullptr, s->d_step, st)) return -2;
    // Q(obs, a) and, in the same kernel, dQ_i/da for both critics (unit output gradient; no critic weight gradients: only the actor
    // optimiser steps here).  The routing of d(-min q)/da to the smaller critic and the 1/B happen in the dy kernel.
    if (b2q_mlp_forward_ex(s->mlp_critic, obs, D, s->cur_a, B, B2Q_MLP_RAW, 0, nullptr, s->q, nullptr, nullptr, nullptr, s->da_c, nullptr, st)) return -2;
    s->launches += 2;
    pdl_launch(k_actor_dy, dim3(B / DY_ROWS), dim3(DY_ROWS * A), 0, st, s->raw_a, eps_cur, s->cur_a, s->cur_logp, s->q, s->da_c, s->da_c + (size_t)B * 16, s->alpha, s->dy_rm, s->dy_bf, s->g_actor + an.ob3, s->losses + 1, B, A, seed * 2, s->d_step);
    if (actor_backward(s, st)) return -2;
  } else {
    return -1;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { s->err = cudaGetErrorString(e); return -2; }
  return 0;
}

int b2q_sac_learn(B2QSacHandle s, const float* obs, const float* act, const float* rew, const float* next_obs, const float* term, const float* eps_next,
                  const float* eps_cur, uint64_t seed, float* losses_out /*device [2]: critic, actor*/, void* stream) {
  if (!s) return -1;
  // the four phases in stream order.  (Running the critics' optimiser step on the side stream beside the actor forward was measured: the two
  // extra cross-stream graph edges cost 7 us more than the 8 us kernel they hide.)
  for (int ph = 0; ph < 4; ph++) {
    int rc = b2q_sac_phase(s, ph, obs, act, rew, next_obs, term, eps_next, eps_cur, seed, stream);
    if (rc) return rc;
  }
  if (losses_out) cudaMemcpyAsync(losses_out, s->losses, 2 * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
  return 0;
}
// Behaviour cloning of a (partial-observation) student from an expert (BC.BClearn, alg/BC.py:53-72): actor step on
// -mean log N(expert_action | mean, std), then critic regression onto the expert's twin Q at the student's fresh sample.
// eps == NULL: the student's sample() draw comes from the counter RNG keyed by `seed` and the device step counter (the key of b2q_sac_learn's
// draws), so the call needs no noise tensor and a CUDA-graph replay draws fresh noise every step.
int b2q_sac_bc_learn_seeded(B2QSacHandle s, const float* obs, const float* ref_obs, int ref_obs_dim, B2QMlpHandle expert_actor, B2QMlpHandle expert_critic,
                            const float* eps, uint64_t seed, float* losses_out, void* stream) {
  if (!s || !obs || !ref_obs || !expert_actor || !expert_critic) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s->B, A = s->A, D = s->D, na = (int)s->an.n, nc = (int)(2 * s->cn.n);
  const Net& an = s->an;
  cudaMemsetAsync(s->losses, 0, 4 * sizeof(float), st);
  cudaMemsetAsync(s->g_actor, 0, (na + nc) * sizeof(float), st);
  s->actor_grad_dirty = true;
  // --- actor
  if (b2q_mlp_forward(expert_actor, ref_obs, ref_obs_dim, nullptr, B, B2Q_MLP_PREDICT, 0, nullptr, s->next_a /*ref action*/, nullptr, nullptr, st)) return -2;
  B2QMlpSaves sa = {nullptr /*x row-major: no consumer*/, s->xa_t, s->ha1_rm, s->ha1_t, s->ha2_rm, s->ha2_t};
  if (b2q_mlp_forward_ex(s->mlp_actor, obs, D, nullptr, B, B2Q_MLP_RAW, 0, nullptr, s->raw_a, nullptr, nullptr, &sa, nullptr, nullptr, st)) return -2;
  pdl_launch(k_bc_dy, dim3(B / DY_ROWS), dim3(DY_ROWS * A), 0, st, s->raw_a, s->next_a, s->dy_rm, s->dy_bf, s->g_actor + an.ob3, s->losses + 1, B, A);
  if (actor_backward(s, st)) return -2;
  pdl_launch(k_adam_pack, dim3((na + 255) / 256), dim3(256), 0, st, s->p_actor, s->g_actor, s->m_a, s->v_a, na, s->lr_a, 0.9f, 0.999f, 1e-8f, s->d_step, (int*)nullptr, dst_of(s, NETS_ACTOR));
  // --- critic: a_now ~ pi_student(obs) (no grad); targets = expert Q(ref_obs, a_now)
  // (the counter still holds the number of completed steps: only the critics' Adam below advances it)
  if (b2q_mlp_forward_ex(s->mlp_actor, obs, D, nullptr, B, B2Q_MLP_SAMPLE, seed, eps, s->cur_a, s->cur_logp, nullptr, nullptr, nullptr,
                         eps ? nullptr : s->d_step, st)) return -2;
  if (b2q_mlp_forward(expert_critic, ref_obs, ref_obs_dim, s->cur_a, B, B2Q_MLP_RAW, 0, nullptr, s->qn, nullptr, nullptr, st)) return -2;
  B2QMlpSaves sv = {nullptr /*x row-major: no consumer*/, s->xc_t, s->hc1_rm, s->hc1_t, s->hc2_rm, s->hc2_t};
  if (b2q_mlp_forward_ex(s->mlp_critic, obs, D, s->cur_a, B, B2Q_MLP_RAW, 0, nullptr, s->q, nullptr, nullptr, &sv, nullptr, nullptr, st)) return -2;
  if (critic_backward(s, st, DqSrc{DQ_TWIN, 0, s->q, nullptr, nullptr, s->qn, nullptr, 0.f, 0.f, s->losses + 0})) return -2;
  // both Adam kernels used step + 1: the critics' closes the step
  pdl_launch(k_adam_pack, dim3((nc + 255) / 256), dim3(256), 0, st, s->p_critic, s->g_critic, s->m_c, s->v_c, nc, s->lr_c, 0.9f, 0.999f, 1e-8f, s->d_step, s->d_step + 1, dst_of(s, NETS_CRITIC));
  s->launches += 10;                                   // the two memsets and the eight kernels launched here (the backward helpers count their own)
  if (losses_out) cudaMemcpyAsync(losses_out, s->losses, 2 * sizeof(float), cudaMemcpyDeviceToDevice, st);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { s->err = cudaGetErrorString(e); return -2; }
  return 0;
}
int b2q_sac_bc_learn(B2QSacHandle s, const float* obs, const float* ref_obs, int ref_obs_dim, B2QMlpHandle expert_actor, B2QMlpHandle expert_critic,
                     const float* eps, float* losses_out, void* stream) {
  if (!eps) return -1;
  return b2q_sac_bc_learn_seeded(s, obs, ref_obs, ref_obs_dim, expert_actor, expert_critic, eps, 0, losses_out, stream);
}
B2QMlpHandle b2q_sac_mlp(B2QSacHandle s, int which) { return !s ? nullptr : (which == 0 ? s->mlp_actor : (which == 1 ? s->mlp_critic : s->mlp_target)); }
float* b2q_sac_grad_ptr(B2QSacHandle s, int which) { return !s ? nullptr : (which == 1 ? s->g_critic : s->g_actor); }   // which == 2: the flat bucket (starts at the actor part)
float* b2q_sac_loss_ptr(B2QSacHandle s) { return s ? s->losses : nullptr; }

int64_t b2q_sac_snapshot_bytes(B2QSacHandle s) { return s ? sac_snapshot_bytes(s) : -1; }
int64_t b2q_sac_snapshot_loss_offset(B2QSacHandle s) {
  if (!s) return -1;
  SacPart parts[8]; sac_parts(s, parts);
  int64_t off = (int64_t)b2q_snap::HDR_BYTES;
  for (int i = 0; parts[i].p != s->losses; i++) off += (int64_t)(parts[i].n * sizeof(float));
  return off;
}
int b2q_sac_snapshot_save(B2QSacHandle s, void* dst, void* stream) {
  if (!s) return -1;
  if (!dst || ((size_t)dst & 15)) { s->err = "b2q_sac_snapshot_save: dst must be a 16-byte aligned device pointer"; return -1; }
  cudaSetDevice(s->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (b2q_snap::write_header(sac_header(s), dst, st) != cudaSuccess) { s->err = "b2q_sac_snapshot_save: header store failed"; return -2; }
  char* o = (char*)dst + b2q_snap::HDR_BYTES;
  SacPart parts[8]; sac_parts(s, parts);
  for (const SacPart& q : parts) { cudaMemcpyAsync(o, q.p, q.n * sizeof(float), cudaMemcpyDeviceToDevice, st); o += q.n * sizeof(float); }
  cudaMemsetAsync(o, 0, 16, st);                     // the tail's padding too: equal learners give equal blobs
  cudaMemcpyAsync(o, s->d_step, 2 * sizeof(int), cudaMemcpyDeviceToDevice, st);
  s->launches++;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { s->err = cudaGetErrorString(e); return -2; }
  return 0;
}
int b2q_sac_snapshot_load(B2QSacHandle s, const void* src, void* stream) {
  if (!s) return -1;
  if (!src || ((size_t)src & 15)) { s->err = "b2q_sac_snapshot_load: src must be a 16-byte aligned device pointer"; return -1; }
  cudaSetDevice(s->device);
  cudaStream_t st = (cudaStream_t)stream;
  // the refusal is a return code, so the header has to reach the host first: one small copy, waited for
  SacSnapHeader got;
  if (cudaMemcpyAsync(&got, src, sizeof got, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
    s->err = "b2q_sac_snapshot_load: header read failed"; return -2;
  }
  const SacSnapHeader mine = sac_header(s);
  if (const char* f = b2q_snap::first_difference(&got, &mine, SAC_SNAP_FIELDS, (int)(sizeof SAC_SNAP_FIELDS / sizeof SAC_SNAP_FIELDS[0]))) {
    s->err = std::string("b2q_sac_snapshot_load: the blob's ") + f + " differs from this learner's";
    return -1;
  }
  const char* o = (const char*)src + b2q_snap::HDR_BYTES;
  SacPart parts[8]; sac_parts(s, parts);
  for (const SacPart& q : parts) { cudaMemcpyAsync(q.p, o, q.n * sizeof(float), cudaMemcpyDeviceToDevice, st); o += q.n * sizeof(float); }
  cudaMemcpyAsync(s->d_step, o, 2 * sizeof(int), cudaMemcpyDeviceToDevice, st);
  // the gradient bucket is not in the blob: every learn clears it before use, and a phase 2 without a phase 0 clears the actor part when
  // this flag is set, so the next step reads the same zeros the saved learner would have
  s->actor_grad_dirty = true;
  return repack_all(s, st);
}


}  // extern "C"
