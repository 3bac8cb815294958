// Tensor-core attention kernels for sm_90a (H100): TMA loads into 128-byte-swizzled shared memory, a two-stage
// mbarrier-tracked ring for the streamed operand, wgmma with FP32 accumulators in registers.
//
//   forward      one CTA = 2 warpgroups = 128 query rows; keys stream in blocks of 128 (D <= 128) or 64 (D <= 256).
//                S = Q K^T (both operands K-major in shared memory), online softmax in registers, O += P V with P taken
//                straight from the S accumulator registers (wgmma A-from-registers) and V as an MN-major operand.
//   backward dQ  one CTA = 128 query rows (D <= 128) or 64 (D <= 256); 64-key blocks.  D = rowsum(dO * O) / sqrt(D) is
//                computed first (and stored for dK/dV), then S = Q K^T, dP = dO V^T, dS = P (dP / sqrt(D) - D),
//                dQ += dS K.
//   backward dKV one CTA = 128 key rows (D <= 128), or 64 key rows whose dK / dV columns are split over the two
//                warpgroups (D <= 256: one warpgroup could not hold both 64 x 256 accumulators); 64-query blocks.
//                S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q.
//
// Operands are 16-bit and row-major with D % 8 == 0 here (kernel.cpp stages anything else); the head dimension is
// padded to 64 / 128 / 256 columns by TMA's zero fill of the out-of-range box columns, rows past R / C are zero-filled
// the same way and masked out of the softmax.  Numerical conventions as in simt_attention.cu: log2-domain running max,
// L = m + log2(l), D pre-scaled by 1/sqrt(D).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "attention_params.h"
#include "backward_common.cuh"
#include "device_state.h"
#include "sm90_ptx.cuh"
#include "tma_host.h"
#include "wgmma.cuh"

namespace mfa {
namespace hop {

using namespace ptx;
using bwd::load_16bit;
using bwd::load_stat;
using bwd::store_stat;

constexpr uint32_t kWG = 128;    // threads per warpgroup
constexpr uint32_t kRows = 64;   // rows of one wgmma M tile (one warpgroup)
constexpr uint32_t kBarBytes = 64;

// Shared-memory tiles are [column chunk][rows][64 16-bit elements], 128-byte swizzled, one TMA box per chunk.
// K-major descriptor of K step kk (16 elements) for the 64-row M / N tile starting at row `row0` of a ROWS-row tile
template <uint32_t ROWS>
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t tile, uint32_t row0, uint32_t kk) {
  return make_smem_desc_sw128(tile + (kk >> 2) * ROWS * 128 + row0 * 128 + (kk & 3) * 32, 16, 1024);
}
// MN-major descriptor: tile rows are the K index, columns the N index; K step kk, N starting at column chunk c0
template <uint32_t ROWS>
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t tile, uint32_t kk, uint32_t c0) {
  return make_smem_desc_sw128(tile + c0 * ROWS * 128 + kk * 16 * 128, ROWS * 128, 1024);
}

template <bool kBF16>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  return kBF16 ? pack_bf16x2(lo, hi) : pack_f16x2(lo, hi);
}
// A-operand fragment of K step kk taken from a 64 x N accumulator (columns 16 kk .. 16 kk + 15)
template <bool kBF16, int NR>
__device__ __forceinline__ void a_frag(const float (&s)[NR], uint32_t kk, uint32_t (&a)[4]) {
  a[0] = pack2<kBF16>(s[8 * kk + 0], s[8 * kk + 1]);
  a[1] = pack2<kBF16>(s[8 * kk + 2], s[8 * kk + 3]);
  a[2] = pack2<kBF16>(s[8 * kk + 4], s[8 * kk + 5]);
  a[3] = pack2<kBF16>(s[8 * kk + 6], s[8 * kk + 7]);
}

__device__ __forceinline__ uint8_t *align1024(uint8_t *p) {
  return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// DCH column chunks of a `rows`-row tile at (column 0, row0, head) -> smem, completion on bar
template <uint32_t DCH, uint32_t ROWS>
__device__ __forceinline__ void load_tile(uint8_t *dst, const CUtensorMap *map, uint64_t *bar, uint32_t row0,
                                          uint32_t head) {
#pragma unroll
  for (uint32_t c = 0; c < DCH; ++c) tma_load_3d(dst + c * ROWS * 128, map, bar, c * 64, row0, head);
}

template <int N>
__device__ __forceinline__ void zero(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) d[i] = 0.f;
}

// FP32 accumulator rows -> global [rows][D] (row-major), columns < D, rows < limit
template <int NR>
__device__ __forceinline__ void store_acc(const float (&acc)[NR], float *out, uint32_t row0, uint32_t limit, uint32_t col0,
                                          uint32_t D, float inv0, float inv1) {
  const uint32_t t = threadIdx.x % kWG;
  const uint32_t r = row0 + (t / 32) * 16 + (t % 32) / 4;
#pragma unroll
  for (int i = 0; i < NR / 4; ++i) {
    const uint32_t col = col0 + 8 * i + 2 * (t % 4);
    if (col >= D) continue;
    if (r < limit)
      *reinterpret_cast<float2 *>(out + static_cast<size_t>(r) * D + col) = make_float2(acc[4 * i] * inv0, acc[4 * i + 1] * inv0);
    if (r + 8 < limit)
      *reinterpret_cast<float2 *>(out + static_cast<size_t>(r + 8) * D + col) =
          make_float2(acc[4 * i + 2] * inv1, acc[4 * i + 3] * inv1);
  }
}

// ================================================================================================ forward
// Split-KV (few query tiles for 132 SMs): the key axis of every tile is cut into `splits` equal ranges handled by
// separate CTAs (blockIdx.z), each leaving a normalised partial O and its log2-sum-exp in the library's workspace,
// laid out [split][head][row].  The partials are merged either by merge_splits (a second launch) or, in the one-launch
// form, by the CTA of each tile that arrives last on the tile's counter.
struct SplitArgs {
  uint32_t blocks_per_split, splits, batch;
  float *O_part, *L_part;  // [split][head][R][D], [split][head][R]
  uint32_t *counters;      // one-launch form: arrivals per (head, tile), returned to zero; nullptr: merged by merge_splits
};

// O[row][4 quad ..] and L[row] from the partials of every split (row = head * R + r)
__device__ __forceinline__ void merge_quad(const SplitArgs &sp, float *O, void *L, int l_prec, uint64_t rows_total,
                                           uint64_t row, uint32_t quad, uint32_t D) {
  float lmax = -INFINITY;
  for (uint32_t s = 0; s < sp.splits; ++s) lmax = fmaxf(lmax, __ldcg(sp.L_part + s * rows_total + row));
  float denom = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (uint32_t s = 0; s < sp.splits; ++s) {
    const float w = exp2f(__ldcg(sp.L_part + s * rows_total + row) - lmax);
    const float4 v = __ldcg(reinterpret_cast<const float4 *>(sp.O_part + (s * rows_total + row) * D) + quad);
    denom += w;
    acc.x = fmaf(w, v.x, acc.x);
    acc.y = fmaf(w, v.y, acc.y);
    acc.z = fmaf(w, v.z, acc.z);
    acc.w = fmaf(w, v.w, acc.w);
  }
  const float inv = 1.0f / denom;
  *reinterpret_cast<float4 *>(O + row * D + 4 * quad) = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
  if (quad == 0) store_stat(L, row, l_prec, lmax + log2f(denom));
}

// second launch of the two-launch form: one thread per (row, 4 columns)
__global__ void __launch_bounds__(128) merge_splits(const SplitArgs sp, float *O, void *L, int l_prec, uint64_t rows_total,
                                                    uint32_t D) {
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t row = idx / (D / 4);
  if (row < rows_total) merge_quad(sp, O, L, l_prec, rows_total, row, static_cast<uint32_t>(idx % (D / 4)), D);
}

template <uint32_t DCH, uint32_t BN>
struct FwdCfg {
  static constexpr uint32_t kThreads = 2 * kWG, kTileM = 2 * kRows;
  static constexpr uint32_t kQBytes = DCH * kTileM * 128, kKVBytes = DCH * BN * 128;
  static constexpr uint32_t kSmemBytes = 1024 + kQBytes + 2 * 2 * kKVBytes + kBarBytes;
};

template <uint32_t DCH, uint32_t BN, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    attention_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                            const __grid_constant__ CUtensorMap mapV, float *__restrict__ O, void *__restrict__ L,
                            uint32_t R, uint32_t C, uint32_t D, float scale_log2, int l_prec, const SplitArgs sp) {
  using Cfg = FwdCfg<DCH, BN>;
  constexpr uint32_t NO = DCH * 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *base = align1024(smem_raw);
  uint8_t *kv = base + Cfg::kQBytes;  // stage s: K at kv + 2 s kKVBytes, V right after it
  uint64_t *bar = reinterpret_cast<uint64_t *>(kv + 4 * Cfg::kKVBytes);  // [0] Q, [1 + s] stage s
  const uint32_t tid = threadIdx.x, wg = tid / kWG, t = tid % kWG;
  const uint32_t head = blockIdx.y, row_base = blockIdx.x * Cfg::kTileM;
  // this CTA's key blocks: [kb0, kb0 + blocks)
  const uint32_t kb0 = blockIdx.z * sp.blocks_per_split;
  const uint32_t blocks = min((C + BN - 1) / BN - kb0, sp.blocks_per_split);

  auto load_kv = [&](uint32_t j, uint32_t s) {
    uint8_t *dst = kv + s * 2 * Cfg::kKVBytes;
    mbar_arrive_expect_tx(&bar[1 + s], 2 * Cfg::kKVBytes);
    load_tile<DCH, BN>(dst, &mapK, &bar[1 + s], (kb0 + j) * BN, head);
    load_tile<DCH, BN>(dst + Cfg::kKVBytes, &mapV, &bar[1 + s], (kb0 + j) * BN, head);
  };
  if (tid == 0) {
    prefetch_tensormap(&mapQ);
    prefetch_tensormap(&mapK);
    prefetch_tensormap(&mapV);
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bar[0], Cfg::kQBytes);
    load_tile<DCH, Cfg::kTileM>(base, &mapQ, &bar[0], row_base, head);
    for (uint32_t s = 0; s < 2 && s < blocks; ++s) load_kv(s, s);
  }

  const uint32_t sQ = smem_u32(base);
  float o[NO / 2];
  zero(o);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  mbar_wait(&bar[0], 0);
  for (uint32_t j = 0; j < blocks; ++j) {
    const uint32_t s = j & 1;
    mbar_wait(&bar[1 + s], (j >> 1) & 1);
    const uint32_t sK = smem_u32(kv + s * 2 * Cfg::kKVBytes), sV = sK + Cfg::kKVBytes;
    float sc[BN / 2];
    zero(sc);
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < DCH * 4; ++kk)
      Wgmma<BN, kBF16>::ss(sc, desc_kmajor<Cfg::kTileM>(sQ, wg * kRows, kk), desc_kmajor<BN>(sK, 0, kk), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sc);

    // keys past C: -inf before the row max
    if ((kb0 + j + 1) * BN > C) {
      const uint32_t c0 = (kb0 + j) * BN + 2 * (t % 4);
#pragma unroll
      for (uint32_t i = 0; i < BN / 8; ++i)
#pragma unroll
        for (uint32_t e = 0; e < 2; ++e)
          if (c0 + 8 * i + e >= C) sc[4 * i + e] = sc[4 * i + 2 + e] = -INFINITY;
    }
    float r0 = -INFINITY, r1 = -INFINITY;
#pragma unroll
    for (uint32_t i = 0; i < BN / 8; ++i) {
      r0 = fmaxf(r0, fmaxf(sc[4 * i], sc[4 * i + 1]));
      r1 = fmaxf(r1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
    }
    r0 = fmaxf(r0, __shfl_xor_sync(0xffffffffu, r0, 1));
    r0 = fmaxf(r0, __shfl_xor_sync(0xffffffffu, r0, 2));
    r1 = fmaxf(r1, __shfl_xor_sync(0xffffffffu, r1, 1));
    r1 = fmaxf(r1, __shfl_xor_sync(0xffffffffu, r1, 2));
    const float mn0 = fmaxf(m0, r0 * scale_log2), mn1 = fmaxf(m1, r1 * scale_log2);
    const float a0 = ex2_approx(m0 - mn0), a1 = ex2_approx(m1 - mn1);  // 0 on the first block (m = -inf)
    m0 = mn0;
    m1 = mn1;
    l0 *= a0;
    l1 *= a1;
#pragma unroll
    for (uint32_t i = 0; i < NO / 8; ++i) {
      o[4 * i] *= a0;
      o[4 * i + 1] *= a0;
      o[4 * i + 2] *= a1;
      o[4 * i + 3] *= a1;
    }
#pragma unroll
    for (uint32_t i = 0; i < BN / 8; ++i) {
      sc[4 * i] = ex2_approx(fmaf(sc[4 * i], scale_log2, -m0));
      sc[4 * i + 1] = ex2_approx(fmaf(sc[4 * i + 1], scale_log2, -m0));
      sc[4 * i + 2] = ex2_approx(fmaf(sc[4 * i + 2], scale_log2, -m1));
      sc[4 * i + 3] = ex2_approx(fmaf(sc[4 * i + 3], scale_log2, -m1));
      l0 += sc[4 * i] + sc[4 * i + 1];
      l1 += sc[4 * i + 2] + sc[4 * i + 3];
    }
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < BN / 16; ++kk) {
      uint32_t a[4];
      a_frag<kBF16>(sc, kk, a);
      Wgmma<NO, kBF16>::rs(o, a, desc_mnmajor<BN>(sV, kk, 0), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncthreads();  // every warpgroup is done with stage s
    if (tid == 0 && j + 2 < blocks) load_kv(j + 2, s);
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const uint32_t row0 = row_base + wg * kRows;
  // unsplit: O and L straight to the caller; split: the normalised partial of this key range
  const size_t slice = static_cast<size_t>(blockIdx.z) * sp.batch + head;
  float *Oout = sp.splits == 1 ? O + static_cast<size_t>(head) * R * D : sp.O_part + slice * R * D;
  store_acc(o, Oout, row0, R, 0, D, 1.0f / l0, 1.0f / l1);
  if (t % 4 == 0) {
    const uint32_t r = row0 + (t / 32) * 16 + (t % 32) / 4;
    void *Lout = sp.splits == 1 ? L : sp.L_part;
    const int prec = sp.splits == 1 ? l_prec : FP32;
    const size_t hb = (sp.splits == 1 ? static_cast<size_t>(head) : slice) * R;
    if (r < R) store_stat(Lout, hb + r, prec, m0 + log2f(l0));
    if (r + 8 < R) store_stat(Lout, hb + r + 8, prec, m1 + log2f(l1));
  }
  if (sp.splits == 1 || sp.counters == nullptr) return;

  // one-launch form: the last CTA of this tile to arrive merges the tile's rows
  __shared__ uint32_t last;
  __threadfence();
  __syncthreads();
  uint32_t *counter = sp.counters + head * gridDim.x + blockIdx.x;
  if (tid == 0) last = atomicAdd(counter, 1u) == sp.splits - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  const uint64_t rows_total = static_cast<uint64_t>(sp.batch) * R;
  for (uint32_t idx = tid; idx < Cfg::kTileM * (D / 4); idx += Cfg::kThreads) {
    const uint32_t r = row_base + idx / (D / 4);
    if (r < R) merge_quad(sp, O, L, l_prec, rows_total, static_cast<uint64_t>(head) * R + r, idx % (D / 4), D);
  }
  if (tid == 0) *counter = 0;
}

// ================================================================================================ backward dQ
template <uint32_t DCH>
struct QCfg {
  static constexpr uint32_t kWarpgroups = DCH == 4 ? 1 : 2;
  static constexpr uint32_t kThreads = kWarpgroups * kWG, kTileM = kWarpgroups * kRows, BN = 64;
  static constexpr uint32_t kQBytes = DCH * kTileM * 128, kKVBytes = DCH * BN * 128;
  static constexpr uint32_t kSmemBytes = 1024 + 2 * kQBytes + 2 * 2 * kKVBytes + kBarBytes;
};

struct BwdArgs {
  const float *O;
  const void *dO;  // for the D term (its memory precision: dO_bf16)
  const void *L;
  void *Dterm;
  float *dQ, *dK, *dV;        // traversal split: partial sums at + blockIdx.z * split_stride
  size_t split_stride;
  uint32_t blocks_per_split;  // traversal blocks per CTA (all of them when unsplit)
  uint32_t R, C, D;
  float scale, scale_log2;
  int l_prec, d_prec, dO_bf16;
};

template <uint32_t DCH, bool kBF16, bool kConvertDO>
__global__ void __launch_bounds__(QCfg<DCH>::kThreads, 1)
    attention_backward_query_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                   const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                   const BwdArgs a) {
  using Cfg = QCfg<DCH>;
  constexpr uint32_t NO = DCH * 64, BN = Cfg::BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *base = align1024(smem_raw);
  uint8_t *kv = base + 2 * Cfg::kQBytes;
  uint64_t *bar = reinterpret_cast<uint64_t *>(kv + 4 * Cfg::kKVBytes);
  const uint32_t tid = threadIdx.x, wg = tid / kWG, t = tid % kWG;
  const uint32_t head = blockIdx.y, row_base = blockIdx.x * Cfg::kTileM;
  const uint32_t kb0 = blockIdx.z * a.blocks_per_split;
  const uint32_t blocks = min((a.C + BN - 1) / BN - kb0, a.blocks_per_split);

  auto load_kv = [&](uint32_t j, uint32_t s) {
    uint8_t *dst = kv + s * 2 * Cfg::kKVBytes;
    mbar_arrive_expect_tx(&bar[1 + s], 2 * Cfg::kKVBytes);
    load_tile<DCH, BN>(dst, &mapK, &bar[1 + s], (kb0 + j) * BN, head);
    load_tile<DCH, BN>(dst + Cfg::kKVBytes, &mapV, &bar[1 + s], (kb0 + j) * BN, head);
  };
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bar[0], 2 * Cfg::kQBytes);
    load_tile<DCH, Cfg::kTileM>(base, &mapQ, &bar[0], row_base, head);
    load_tile<DCH, Cfg::kTileM>(base + Cfg::kQBytes, &mapdO, &bar[0], row_base, head);
    for (uint32_t s = 0; s < 2 && s < blocks; ++s) load_kv(s, s);
  }

  // D = rowsum(dO * O) / sqrt(D) for this thread's two rows (the four threads of a row split the columns), while the
  // tiles are in flight; stored for the dK/dV kernel, kept in FP32 here
  const uint32_t row0 = row_base + wg * kRows;
  const uint32_t r = row0 + (t / 32) * 16 + (t % 32) / 4;
  const size_t hb = static_cast<size_t>(head) * a.R;
  float Dr[2], Lr[2];
#pragma unroll
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t rc = min(r + 8 * h, a.R - 1);
    const float *Orow = a.O + (hb + rc) * a.D;
    const size_t drow = (hb + rc) * a.D;
    float part = 0.f;
    for (uint32_t d = 2 * (t % 4); d < a.D; d += 8) {
      const float2 ov = *reinterpret_cast<const float2 *>(Orow + d);
      part = fmaf(ov.x, load_16bit(a.dO, drow + d, a.dO_bf16), part);
      part = fmaf(ov.y, load_16bit(a.dO, drow + d + 1, a.dO_bf16), part);
    }
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 2);
    Dr[h] = part * a.scale;
    Lr[h] = load_stat(a.L, hb + rc, a.l_prec);
    if (t % 4 == 0 && r + 8 * h < a.R && blockIdx.z == 0) store_stat(a.Dterm, hb + r + 8 * h, a.d_prec, Dr[h]);
  }

  const uint32_t sQ = smem_u32(base), sdO = sQ + Cfg::kQBytes;
  mbar_wait(&bar[0], 0);
  if constexpr (kConvertDO) {
    // BF16 dO beside FP16 Q/K/V: wgmma takes one element type for A and B, so the resident dO tile is rewritten as
    // FP16 in place (exact for 2^-14 <= |x| < 65504)
    uint4 *tile = reinterpret_cast<uint4 *>(base + Cfg::kQBytes);
    for (uint32_t i = tid; i < Cfg::kQBytes / 16; i += Cfg::kThreads) tile[i] = bwd::bf16x8_to_f16x8(tile[i]);
    fence_proxy_async_smem();
    __syncthreads();
  }
  float dq[NO / 2];
  zero(dq);
  for (uint32_t j = 0; j < blocks; ++j) {
    const uint32_t s = j & 1;
    mbar_wait(&bar[1 + s], (j >> 1) & 1);
    const uint32_t sK = smem_u32(kv + s * 2 * Cfg::kKVBytes), sV = sK + Cfg::kKVBytes;
    float sc[BN / 2], dp[BN / 2];
    zero(sc);
    zero(dp);
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < DCH * 4; ++kk)
      Wgmma<BN, kBF16>::ss(sc, desc_kmajor<Cfg::kTileM>(sQ, wg * kRows, kk), desc_kmajor<BN>(sK, 0, kk), kk > 0);
#pragma unroll
    for (uint32_t kk = 0; kk < DCH * 4; ++kk)
      Wgmma<BN, kBF16>::ss(dp, desc_kmajor<Cfg::kTileM>(sdO, wg * kRows, kk), desc_kmajor<BN>(sV, 0, kk), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sc);
    fence_regs(dp);
    const uint32_t c0 = (kb0 + j) * BN + 2 * (t % 4);
#pragma unroll
    for (uint32_t i = 0; i < BN / 8; ++i)
#pragma unroll
      for (uint32_t e = 0; e < 4; ++e) {
        const uint32_t h = e >> 1, k = 4 * i + e;
        const float p = c0 + 8 * i + (e & 1) < a.C ? ex2_approx(fmaf(sc[k], a.scale_log2, -Lr[h])) : 0.f;
        sc[k] = p * fmaf(dp[k], a.scale, -Dr[h]);  // dS
      }
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < BN / 16; ++kk) {
      uint32_t f[4];
      a_frag<kBF16>(sc, kk, f);
      Wgmma<NO, kBF16>::rs(dq, f, desc_mnmajor<BN>(sK, kk, 0), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dq);
    __syncthreads();
    if (tid == 0 && j + 2 < blocks) load_kv(j + 2, s);
  }
  store_acc(dq, a.dQ + blockIdx.z * a.split_stride + hb * a.D, row0, a.R, 0, a.D, 1.f, 1.f);
}

// ================================================================================================ backward dK/dV
template <uint32_t DCH>
struct KVCfg {
  static constexpr bool kSplitD = DCH == 4;  // both warpgroups on the same 64 keys, half of the D columns each
  static constexpr uint32_t kThreads = 2 * kWG, kTileN = kSplitD ? kRows : 2 * kRows, BM = 64;
  static constexpr uint32_t kAcc = kSplitD ? 128 : DCH * 64;  // accumulator columns per warpgroup
  static constexpr uint32_t kKBytes = DCH * kTileN * 128, kQBytes = DCH * BM * 128;
  static constexpr uint32_t kSmemBytes = 1024 + 2 * kKBytes + 2 * 2 * kQBytes + kBarBytes;
};

template <uint32_t DCH, bool kBF16, bool kConvertDO>
__global__ void __launch_bounds__(2 * kWG, 1)
    attention_backward_key_value_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                       const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                       const BwdArgs a) {
  using Cfg = KVCfg<DCH>;
  constexpr uint32_t BM = Cfg::BM, NA = Cfg::kAcc;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *base = align1024(smem_raw);
  uint8_t *qd = base + 2 * Cfg::kKBytes;  // stage s: Q at qd + 2 s kQBytes, dO right after it
  uint64_t *bar = reinterpret_cast<uint64_t *>(qd + 4 * Cfg::kQBytes);
  const uint32_t tid = threadIdx.x, wg = tid / kWG, t = tid % kWG;
  const uint32_t head = blockIdx.y, key_base = blockIdx.x * Cfg::kTileN;
  const uint32_t qb0 = blockIdx.z * a.blocks_per_split;
  const uint32_t blocks = min((a.R + BM - 1) / BM - qb0, a.blocks_per_split);

  auto load_qd = [&](uint32_t i, uint32_t s) {
    uint8_t *dst = qd + s * 2 * Cfg::kQBytes;
    mbar_arrive_expect_tx(&bar[1 + s], 2 * Cfg::kQBytes);
    load_tile<DCH, BM>(dst, &mapQ, &bar[1 + s], (qb0 + i) * BM, head);
    load_tile<DCH, BM>(dst + Cfg::kQBytes, &mapdO, &bar[1 + s], (qb0 + i) * BM, head);
  };
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bar[0], 2 * Cfg::kKBytes);
    load_tile<DCH, Cfg::kTileN>(base, &mapK, &bar[0], key_base, head);
    load_tile<DCH, Cfg::kTileN>(base + Cfg::kKBytes, &mapV, &bar[0], key_base, head);
    for (uint32_t s = 0; s < 2 && s < blocks; ++s) load_qd(s, s);
  }
  const uint32_t sK = smem_u32(base), sV = sK + Cfg::kKBytes;
  const uint32_t krow = Cfg::kSplitD ? 0 : wg * kRows;      // this warpgroup's key rows inside the tile
  const uint32_t nchunk = Cfg::kSplitD ? wg * (NA / 64) : 0;  // ... and its first accumulator column chunk
  const size_t hb = static_cast<size_t>(head) * a.R;
  float dv[NA / 2], dk[NA / 2];
  zero(dv);
  zero(dk);
  mbar_wait(&bar[0], 0);
  for (uint32_t i = 0; i < blocks; ++i) {
    const uint32_t s = i & 1;
    // per-query statistics of this thread's 16 columns, loaded while the tiles land
    float Lq[BM / 4], Dq[BM / 4];
    const uint32_t q0 = (qb0 + i) * BM + 2 * (t % 4);
#pragma unroll
    for (uint32_t j = 0; j < BM / 8; ++j)
#pragma unroll
      for (uint32_t e = 0; e < 2; ++e) {
        const uint32_t q = min(q0 + 8 * j + e, a.R - 1);
        Lq[2 * j + e] = load_stat(a.L, hb + q, a.l_prec);
        Dq[2 * j + e] = load_stat(a.Dterm, hb + q, a.d_prec);
      }
    mbar_wait(&bar[1 + s], (i >> 1) & 1);
    if constexpr (kConvertDO) {
      // BF16 dO beside FP16 Q/K/V on a small grid: the streamed dO tile is rewritten as FP16 in place (a grid of more
      // than one wave converts dO once, in a pass of its own, instead)
      uint4 *tile = reinterpret_cast<uint4 *>(qd + s * 2 * Cfg::kQBytes + Cfg::kQBytes);
      for (uint32_t k = tid; k < Cfg::kQBytes / 16; k += Cfg::kThreads) tile[k] = bwd::bf16x8_to_f16x8(tile[k]);
      fence_proxy_async_smem();
      __syncthreads();
    }
    const uint32_t sQ = smem_u32(qd + s * 2 * Cfg::kQBytes), sdO = sQ + Cfg::kQBytes;
    float st[BM / 2], dpt[BM / 2];
    zero(st);
    zero(dpt);
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < DCH * 4; ++kk)
      Wgmma<BM, kBF16>::ss(st, desc_kmajor<Cfg::kTileN>(sK, krow, kk), desc_kmajor<BM>(sQ, 0, kk), kk > 0);
#pragma unroll
    for (uint32_t kk = 0; kk < DCH * 4; ++kk)
      Wgmma<BM, kBF16>::ss(dpt, desc_kmajor<Cfg::kTileN>(sV, krow, kk), desc_kmajor<BM>(sdO, 0, kk), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(st);
    fence_regs(dpt);
#pragma unroll
    for (uint32_t j = 0; j < BM / 8; ++j)
#pragma unroll
      for (uint32_t e = 0; e < 4; ++e) {
        const uint32_t k = 4 * j + e, c = 2 * j + (e & 1);
        const float p = q0 + 8 * j + (e & 1) < a.R ? ex2_approx(fmaf(st[k], a.scale_log2, -Lq[c])) : 0.f;
        st[k] = p;                                  // P^T
        dpt[k] = p * fmaf(dpt[k], a.scale, -Dq[c]);  // dS^T
      }
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < BM / 16; ++kk) {
      uint32_t f[4];
      a_frag<kBF16>(st, kk, f);
      Wgmma<NA, kBF16>::rs(dv, f, desc_mnmajor<BM>(sdO, kk, nchunk), 1);
      a_frag<kBF16>(dpt, kk, f);
      Wgmma<NA, kBF16>::rs(dk, f, desc_mnmajor<BM>(sQ, kk, nchunk), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dv);
    fence_regs(dk);
    __syncthreads();
    if (tid == 0 && i + 2 < blocks) load_qd(i + 2, s);
  }
  const size_t kb = static_cast<size_t>(head) * a.C * a.D;
  const uint32_t row0 = key_base + krow, col0 = nchunk * 64;
  store_acc(dv, a.dV + blockIdx.z * a.split_stride + kb, row0, a.C, col0, a.D, 1.f, 1.f);
  store_acc(dk, a.dK + blockIdx.z * a.split_stride + kb, row0, a.C, col0, a.D, 1.f, 1.f);
}

static uint32_t chunks(uint32_t D) { return D <= 64 ? 1 : (D <= 128 ? 2 : 4); }

// ================================================================================================ split merges
// out[t][i] = sum_s part[s][t][i] (t = tensor: dQ, or dV and dK); the backward needs no re-normalisation across splits
// (L and D are inputs), so this is a plain, deterministic sum
__global__ void __launch_bounds__(256) sum_splits(const float4 *__restrict__ part, float4 *__restrict__ out0,
                                                  float4 *__restrict__ out1, size_t quads, size_t split_stride_quads,
                                                  uint32_t splits) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= quads) return;
  const float4 *src = part + blockIdx.y * quads + i;
  float4 acc = __ldcg(src);
  for (uint32_t s = 1; s < splits; ++s) {
    const float4 v = __ldcg(src + s * split_stride_quads);
    acc.x += v.x;
    acc.y += v.y;
    acc.z += v.z;
    acc.w += v.w;
  }
  (blockIdx.y == 0 ? out0 : out1)[i] = acc;
}

// How many equal key ranges to cut every forward tile into: only when the SMs would otherwise idle, only into ranges
// of at least `min_blocks` key blocks (min_blocks and max_splits are the parameter-table row's tuning columns;
// min_blocks = 0 turns splitting off)
static uint32_t choose_splits(uint32_t items, uint32_t total_blocks, uint32_t sm_count, uint32_t min_blocks,
                              uint32_t max_splits) {
  if (items * 2 > sm_count || min_blocks == 0) return 1;
  if (max_splits > 16) max_splits = 16;
  const uint32_t target = sm_count / items;
  uint32_t best = 1;
  for (uint32_t s = 2; s <= target && s <= max_splits; ++s)
    if (total_blocks % s == 0 && total_blocks / s >= min_blocks) best = s;
  return best;
}

// Traversal blocks per CTA of a backward kernel: all of them, or (few CTAs for the SMs) ranges of at least min_blocks,
// at most max_splits (<= 8) ranges
static uint32_t choose_blocks_per_split(uint32_t ctas, uint32_t total_blocks, uint32_t sm_count, uint32_t min_blocks,
                                        uint32_t max_splits) {
  if (ctas * 2 > sm_count || min_blocks == 0 || total_blocks < 2 * min_blocks) return total_blocks;
  if (max_splits > 8) max_splits = 8;
  uint32_t splits = sm_count / ctas;
  if (splits > max_splits) splits = max_splits;
  if (splits < 2) return total_blocks;
  uint32_t per = (total_blocks + splits - 1) / splits;
  if (per < min_blocks) per = min_blocks;
  return per;
}

static int g_forward_fused = 0;  // split-KV merge: 0 = merge_splits launch, 1 = inside the attention kernel

// ================================================================================================ launchers
template <typename Kernel>
static cudaError_t prepare(Kernel kernel, uint32_t smem) {
  return ensure_max_dynamic_smem(reinterpret_cast<const void *>(kernel), smem, current_device());
}

template <uint32_t DCH, uint32_t BN, bool kBF16>
cudaError_t launch_forward(const AttentionParams &p, cudaStream_t stream) {
  using Cfg = FwdCfg<DCH, BN>;
  auto kernel = attention_forward_wgmma<DCH, BN, kBF16>;
  cudaError_t e;
  if ((e = prepare(kernel, Cfg::kSmemBytes)) != cudaSuccess) return e;
  CUtensorMap mapQ, mapK, mapV;
  if ((e = make_tensor_map_16bit(&mapQ, p.buf[sQ], p.R, p.D, p.batch, Cfg::kTileM)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapK, p.buf[sK], p.C, p.D, p.batch, BN)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapV, p.buf[sV], p.C, p.D, p.batch, BN)) != cudaSuccess) return e;
  const int device = current_device();
  const uint32_t tiles = (p.R + Cfg::kTileM - 1) / Cfg::kTileM, total_blocks = (p.C + BN - 1) / BN;
  const uint32_t splits = choose_splits(tiles * p.batch, total_blocks, device_sm_count(device), p.split_min_blocks, p.split_max);
  SplitArgs sp{total_blocks / splits, splits, p.batch, nullptr, nullptr, nullptr};
  const uint64_t rows_total = static_cast<uint64_t>(p.batch) * p.R;
  if (splits > 1) {
    void *ws = nullptr;
    const size_t o_elems = splits * rows_total * p.D;
    if ((e = workspace_for(device, stream, (o_elems + splits * rows_total) * sizeof(float), &ws)) != cudaSuccess) return e;
    sp.O_part = reinterpret_cast<float *>(static_cast<char *>(ws) + kWorkspaceCounterBytes);
    sp.L_part = sp.O_part + o_elems;
    if (g_forward_fused && tiles * p.batch * sizeof(uint32_t) <= kWorkspaceCounterBytes) sp.counters = static_cast<uint32_t *>(ws);
  }
  const dim3 grid(tiles, p.batch, splits);
  kernel<<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(mapQ, mapK, mapV, static_cast<float *>(p.buf[sO]), p.buf[sL],
                                                           p.R, p.C, p.D, p.scale_log2, p.prec[sL], sp);
  if ((e = cudaGetLastError()) != cudaSuccess || splits == 1 || sp.counters) return e;
  const uint64_t threads = rows_total * (p.D / 4);
  merge_splits<<<static_cast<uint32_t>((threads + 127) / 128), 128, 0, stream>>>(sp, static_cast<float *>(p.buf[sO]),
                                                                                 p.buf[sL], p.prec[sL], rows_total, p.D);
  return cudaGetLastError();
}

// partial accumulators of a traversal split in the workspace: [split][tensor][batch][rows][D] FP32
static cudaError_t split_scratch(BwdArgs &a, uint32_t splits, uint32_t tensors, size_t tensor_elems, cudaStream_t stream,
                                 float **scratch) {
  void *ws = nullptr;
  cudaError_t e = workspace_for(current_device(), stream, splits * tensors * tensor_elems * sizeof(float), &ws);
  if (e != cudaSuccess) return e;
  *scratch = reinterpret_cast<float *>(static_cast<char *>(ws) + kWorkspaceCounterBytes);
  a.split_stride = tensors * tensor_elems;
  return cudaSuccess;
}

static cudaError_t launch_sum(const float *scratch, float *out0, float *out1, size_t tensor_elems, uint32_t tensors,
                              size_t split_stride, uint32_t splits, cudaStream_t stream) {
  const size_t quads = tensor_elems / 4;  // D % 8 == 0
  sum_splits<<<dim3(static_cast<uint32_t>((quads + 255) / 256), tensors), 256, 0, stream>>>(
      reinterpret_cast<const float4 *>(scratch), reinterpret_cast<float4 *>(out0), reinterpret_cast<float4 *>(out1), quads,
      split_stride / 4, splits);
  return cudaGetLastError();
}

static BwdArgs backward_args(const AttentionParams &p) {
  BwdArgs a;
  a.O = static_cast<const float *>(p.buf[sO]);
  a.dO = p.buf[sdO];
  a.L = p.buf[sL];
  a.Dterm = p.buf[sD];
  a.dQ = static_cast<float *>(p.buf[sdQ]);
  a.dK = static_cast<float *>(p.buf[sdK]);
  a.dV = static_cast<float *>(p.buf[sdV]);
  a.R = p.R;
  a.C = p.C;
  a.D = p.D;
  a.scale = p.scale;
  a.scale_log2 = p.scale_log2;
  a.l_prec = p.prec[sL];
  a.d_prec = p.prec[sD];
  a.dO_bf16 = p.prec[sdO] == BF16;
  return a;
}

template <uint32_t DCH, bool kBF16, bool kConvertDO>
cudaError_t launch_query(const AttentionParams &p, cudaStream_t stream) {
  using Cfg = QCfg<DCH>;
  auto kernel = attention_backward_query_wgmma<DCH, kBF16, kConvertDO>;
  cudaError_t e;
  if ((e = prepare(kernel, Cfg::kSmemBytes)) != cudaSuccess) return e;
  CUtensorMap mapQ, mapdO, mapK, mapV;
  if ((e = make_tensor_map_16bit(&mapQ, p.buf[sQ], p.R, p.D, p.batch, Cfg::kTileM)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapdO, p.buf[sdO], p.R, p.D, p.batch, Cfg::kTileM)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapK, p.buf[sK], p.C, p.D, p.batch, Cfg::BN)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapV, p.buf[sV], p.C, p.D, p.batch, Cfg::BN)) != cudaSuccess) return e;
  BwdArgs a = backward_args(p);
  const uint32_t tiles = (p.R + Cfg::kTileM - 1) / Cfg::kTileM, total_blocks = (p.C + Cfg::BN - 1) / Cfg::BN;
  a.blocks_per_split = choose_blocks_per_split(tiles * p.batch, total_blocks, device_sm_count(current_device()),
                                               p.split_min_blocks, p.split_max);
  const uint32_t splits = (total_blocks + a.blocks_per_split - 1) / a.blocks_per_split;
  const size_t tensor_elems = static_cast<size_t>(p.batch) * p.R * p.D;
  float *scratch = nullptr;
  if (splits > 1) {
    if ((e = split_scratch(a, splits, 1, tensor_elems, stream, &scratch)) != cudaSuccess) return e;
    a.dQ = scratch;
  }
  kernel<<<dim3(tiles, p.batch, splits), Cfg::kThreads, Cfg::kSmemBytes, stream>>>(mapQ, mapdO, mapK, mapV, a);
  if ((e = cudaGetLastError()) != cudaSuccess || splits == 1) return e;
  return launch_sum(scratch, static_cast<float *>(p.buf[sdQ]), nullptr, tensor_elems, 1, a.split_stride, splits, stream);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO>
cudaError_t launch_key_value(const AttentionParams &p, cudaStream_t stream) {
  using Cfg = KVCfg<DCH>;
  auto kernel = attention_backward_key_value_wgmma<DCH, kBF16, kConvertDO>;
  cudaError_t e;
  if ((e = prepare(kernel, Cfg::kSmemBytes)) != cudaSuccess) return e;
  CUtensorMap mapQ, mapdO, mapK, mapV;
  if ((e = make_tensor_map_16bit(&mapQ, p.buf[sQ], p.R, p.D, p.batch, Cfg::BM)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapdO, p.buf[sdO], p.R, p.D, p.batch, Cfg::BM)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapK, p.buf[sK], p.C, p.D, p.batch, Cfg::kTileN)) != cudaSuccess) return e;
  if ((e = make_tensor_map_16bit(&mapV, p.buf[sV], p.C, p.D, p.batch, Cfg::kTileN)) != cudaSuccess) return e;
  BwdArgs a = backward_args(p);
  const uint32_t tiles = (p.C + Cfg::kTileN - 1) / Cfg::kTileN, total_blocks = (p.R + Cfg::BM - 1) / Cfg::BM;
  a.blocks_per_split = choose_blocks_per_split(tiles * p.batch, total_blocks, device_sm_count(current_device()),
                                               p.split_min_blocks, p.split_max);
  const uint32_t splits = (total_blocks + a.blocks_per_split - 1) / a.blocks_per_split;
  const size_t tensor_elems = static_cast<size_t>(p.batch) * p.C * p.D;
  float *scratch = nullptr;
  if (splits > 1) {
    if ((e = split_scratch(a, splits, 2, tensor_elems, stream, &scratch)) != cudaSuccess) return e;
    a.dV = scratch;
    a.dK = scratch + tensor_elems;
  }
  kernel<<<dim3(tiles, p.batch, splits), Cfg::kThreads, Cfg::kSmemBytes, stream>>>(mapQ, mapdO, mapK, mapV, a);
  if ((e = cudaGetLastError()) != cudaSuccess || splits == 1) return e;
  return launch_sum(scratch, static_cast<float *>(p.buf[sdV]), static_cast<float *>(p.buf[sdK]), tensor_elems, 2,
                    a.split_stride, splits, stream);
}

// dK/dV with BF16 dO beside FP16 Q/K/V: a grid of more than one wave converts dO once, in a pass of its own
static bool key_value_converts_dO_first(uint32_t C, uint32_t D, uint32_t batch) {
  const uint32_t tile = chunks(D) == 4 ? KVCfg<4>::kTileN : KVCfg<1>::kTileN;
  return static_cast<uint64_t>((C + tile - 1) / tile) * batch > device_sm_count(current_device());
}

}  // namespace hop

void tcgen05_forward_set_fused(int enabled) { hop::g_forward_fused = enabled; }

uint32_t tcgen05_forward_max_head() { return 256; }
uint32_t tcgen05_backward_max_head() { return 256; }

// Transposed operands are staged row-major by kernel.cpp; the descriptor heuristic keeps the shapes whose transposed
// view has a 16-byte row pitch (sequence length % 8 == 0) on the tensor cores, as it always has.
bool tcgen05_forward_transposes_ok(uint32_t R, uint32_t C, bool tQ, bool tK, bool tV) {
  return (!tQ || R % 8 == 0) && (!tK || C % 8 == 0) && (!tV || C % 8 == 0);
}
bool tcgen05_backward_transposes_ok(uint32_t R, uint32_t C, bool tQ, bool tK, bool tV, bool tO) {
  return (!tQ || R % 8 == 0) && (!tK || C % 8 == 0) && (!tV || C % 8 == 0) && (!tO || R % 8 == 0);
}

static bool row_major_16bit(const AttentionParams &p) {
  for (int s = 0; s < kSlots; ++s)
    if (p.transposed[s]) return false;
  return (p.prec[sQ] == FP16 || p.prec[sQ] == BF16) && p.prec[sK] == p.prec[sQ] && p.prec[sV] == p.prec[sQ] &&
         p.D % 8 == 0 && p.D <= 256;
}

cudaError_t launch_tcgen05_forward(const AttentionParams &p, cudaStream_t stream) {
  if (!row_major_16bit(p) || p.prec[sO] != FP32) {
    set_launch_detail("descriptor is outside the wgmma forward kernel's domain");
    return cudaErrorInvalidValue;
  }
  const bool bf16 = p.prec[sQ] == BF16;
  switch (hop::chunks(p.D)) {
    case 1: return bf16 ? hop::launch_forward<1, 128, true>(p, stream) : hop::launch_forward<1, 128, false>(p, stream);
    case 2: return bf16 ? hop::launch_forward<2, 128, true>(p, stream) : hop::launch_forward<2, 128, false>(p, stream);
    default: return bf16 ? hop::launch_forward<4, 64, true>(p, stream) : hop::launch_forward<4, 64, false>(p, stream);
  }
}

static bool backward_ok(const AttentionParams &p) {
  const bool dO_ok = p.prec[sdO] == p.prec[sQ] || (p.prec[sQ] == FP16 && p.prec[sdO] == BF16);
  return row_major_16bit(p) && dO_ok && p.prec[sO] == FP32 && p.prec[sdQ] == FP32 && p.prec[sdK] == FP32 &&
         p.prec[sdV] == FP32;
}

cudaError_t launch_tcgen05_backward_query(const AttentionParams &p, cudaStream_t stream) {
  if (!backward_ok(p)) {
    set_launch_detail("descriptor is outside the wgmma backward kernels' domain");
    return cudaErrorInvalidValue;
  }
  const bool bf16 = p.prec[sQ] == BF16, convert = p.prec[sdO] != p.prec[sQ];
#define MFA_Q_DISPATCH(DCH_)                                                     \
  if (convert) return hop::launch_query<DCH_, false, true>(p, stream);          \
  return bf16 ? hop::launch_query<DCH_, true, false>(p, stream) : hop::launch_query<DCH_, false, false>(p, stream);
  switch (hop::chunks(p.D)) {
    case 1: { MFA_Q_DISPATCH(1) }
    case 2: { MFA_Q_DISPATCH(2) }
    default: { MFA_Q_DISPATCH(4) }
  }
#undef MFA_Q_DISPATCH
}

cudaError_t launch_tcgen05_backward_key_value(const AttentionParams &p, cudaStream_t stream) {
  if (!backward_ok(p)) {
    set_launch_detail("descriptor is outside the wgmma backward kernels' domain");
    return cudaErrorInvalidValue;
  }
  const bool convert = p.prec[sdO] != p.prec[sQ];
  if (convert && hop::key_value_converts_dO_first(p.C, p.D, p.batch)) {
    AttentionParams q = p;
    const uint64_t elements = static_cast<uint64_t>(p.batch) * p.R * p.D;
    void *ws = nullptr;
    cudaError_t e = workspace_for(current_device(), stream, elements * 2, &ws, /*slot=*/2);
    if (e != cudaSuccess) return e;
    void *converted = static_cast<char *>(ws) + kWorkspaceCounterBytes;
    if ((e = launch_bf16_to_f16(p.buf[sdO], converted, elements, stream)) != cudaSuccess) return e;
    q.buf[sdO] = converted;
    q.prec[sdO] = q.prec[sQ];
    return launch_tcgen05_backward_key_value(q, stream);
  }
  const bool bf16 = p.prec[sQ] == BF16;
#define MFA_KV_DISPATCH(DCH_)                                                    \
  if (convert) return hop::launch_key_value<DCH_, false, true>(p, stream);      \
  return bf16 ? hop::launch_key_value<DCH_, true, false>(p, stream) : hop::launch_key_value<DCH_, false, false>(p, stream);
  switch (hop::chunks(p.D)) {
    case 1: { MFA_KV_DISPATCH(1) }
    case 2: { MFA_KV_DISPATCH(2) }
    default: { MFA_KV_DISPATCH(4) }
  }
#undef MFA_KV_DISPATCH
}

// 1 launch, or 2 (attention + merge_splits) when split-KV engages with the two-launch merge
uint32_t tcgen05_forward_launch_count(uint32_t R, uint32_t C, uint32_t D, uint32_t batch, uint32_t min_blocks,
                                      uint32_t max_splits) {
  const uint32_t bn = hop::chunks(D) == 4 ? 64 : 128, tiles = (R + 127) / 128;
  const uint32_t splits =
      hop::choose_splits(tiles * batch, (C + bn - 1) / bn, device_sm_count(current_device()), min_blocks, max_splits);
  return splits > 1 && !(hop::g_forward_fused && tiles * batch * sizeof(uint32_t) <= kWorkspaceCounterBytes) ? 2 : 1;
}

// kernel (+ sum_splits when the traversal split engages) (+ the dO conversion pass of dK/dV on large grids)
uint32_t tcgen05_backward_launch_count(int type, uint32_t R, uint32_t C, uint32_t D, uint32_t batch, uint32_t min_blocks,
                                       uint32_t max_splits, bool convert_dO) {
  const bool key_value = type == 2;  // MFA_BACKWARD_KEY_VALUE
  uint32_t threads, smem, par, trav, head;
  tcgen05_backward_geometry(type, D, &threads, &smem, &par, &trav, &head);
  const uint32_t tiles = ((key_value ? C : R) + par - 1) / par, total = ((key_value ? R : C) + trav - 1) / trav;
  const uint32_t per = hop::choose_blocks_per_split(tiles * batch, total, device_sm_count(current_device()), min_blocks, max_splits);
  return (per < total ? 2 : 1) + (key_value && convert_dO && hop::key_value_converts_dO_first(C, D, batch) ? 1 : 0);
}

void tcgen05_forward_geometry(uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par, uint32_t *trav,
                              uint32_t *head) {
  const uint32_t c = hop::chunks(D);
  *threads = hop::FwdCfg<1, 128>::kThreads;
  *smem_bytes = c == 1 ? hop::FwdCfg<1, 128>::kSmemBytes
                       : (c == 2 ? hop::FwdCfg<2, 128>::kSmemBytes : hop::FwdCfg<4, 64>::kSmemBytes);
  *par = hop::FwdCfg<1, 128>::kTileM;
  *trav = c == 4 ? 64 : 128;
  const uint32_t padded = (D + 7) / 8 * 8;
  *head = c * 64 < padded ? c * 64 : padded;
}

void tcgen05_backward_geometry(int type, uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par,
                               uint32_t *trav, uint32_t *head) {
  const uint32_t c = hop::chunks(D);
  if (type == 1) {  // MFA_BACKWARD_QUERY
    *threads = c == 4 ? hop::QCfg<4>::kThreads : hop::QCfg<1>::kThreads;
    *smem_bytes = c == 1 ? hop::QCfg<1>::kSmemBytes : (c == 2 ? hop::QCfg<2>::kSmemBytes : hop::QCfg<4>::kSmemBytes);
    *par = c == 4 ? hop::QCfg<4>::kTileM : hop::QCfg<1>::kTileM;
    *trav = hop::QCfg<1>::BN;
  } else {
    *threads = hop::KVCfg<1>::kThreads;
    *smem_bytes = c == 1 ? hop::KVCfg<1>::kSmemBytes : (c == 2 ? hop::KVCfg<2>::kSmemBytes : hop::KVCfg<4>::kSmemBytes);
    *par = c == 4 ? hop::KVCfg<4>::kTileN : hop::KVCfg<1>::kTileN;
    *trav = hop::KVCfg<1>::BM;
  }
  const uint32_t padded = (D + 7) / 8 * 8;
  *head = c * 64 < padded ? c * 64 : padded;
}

}  // namespace mfa
