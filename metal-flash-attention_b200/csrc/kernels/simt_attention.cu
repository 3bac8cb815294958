// SIMT FP32 attention kernels for sm_90a: forward, backward-dQ, backward-dK/dV.
//
// This family is the H100 counterpart of the reference's FP32 code path: every contraction is an
// FP32 FMA on the CUDA cores (the reference's FP32 simdgroup_matrix MMAs are ALU FMAs as well), so
// results meet the reference's FP32 tolerance (2e-5 absolute, SquareAttentionTest.swift:547-554).
// It accepts everything the reference's API accepts: any R, C, any D <= 512, per-operand
// transposes, FP32/FP16/BF16 memory precisions.  The tensor-core family in
// wgmma_attention.cu covers the 16-bit hot path.
//
// Algorithm follows the reference kernels' structure, not their code:
//   forward         loopForward           AttentionKernel+Source.swift:158-200
//   backward dQ     loopBackwardQuery     AttentionKernel+Source.swift:202-242, computeD +Softmax.swift:32-221
//   backward dK/dV  loopBackwardKeyValue  AttentionKernel+Source.swift:244-293
// Numerical conventions: log2-domain running max m, L = m + log2(l),
// D stored pre-scaled by 1/sqrt(D), BF16 stores truncate, edge columns masked before softmax.
//
// Tiling: one CTA = 256 threads = a 64 x 64 block of the attention matrix; thread (tx, ty) owns
// the 4 x 4 patch {rows ty+16i} x {cols tx+16j}.  Operands are staged through shared memory as
// FP32 in 64 x 32 (contraction over D) and 64 x 64 (accumulation) tiles; output accumulators
// (64 x D) live in registers, 4 rows x (D/16) columns per thread.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include "attention_params.h"

namespace mfa {
namespace simt {

constexpr int kThreads = 256;
constexpr int kBlock = 64;      // rows and columns of the attention-matrix block
constexpr int kDC = 32;         // head-dimension chunk for the "outer product" contractions
constexpr int kLDA = kDC + 4;   // padded leading dimension of 64 x 32 tiles (float4-aligned, conflict-free)
constexpr int kLDP = kBlock + 4;  // padded leading dimension of 64 x 64 tiles
constexpr int kSmemFloats = 2 * kBlock * kLDA + 2 * kBlock * kLDP;
constexpr int kSmemBytes = kSmemFloats * 4;

struct Operand {
  const void *ptr;
  uint32_t seq;  // sequence length of this operand (R or C)
  uint32_t D;
  int prec;
  int transposed;
};

__device__ __forceinline__ float load_elem(const void *p, size_t i, int prec) {
  if (prec == FP32) return reinterpret_cast<const float *>(p)[i];
  uint16_t h = reinterpret_cast<const uint16_t *>(p)[i];
  if (prec == FP16) return __half2float(__ushort_as_half(h));
  return __uint_as_float(static_cast<uint32_t>(h) << 16);  // BF16 -> FP32 is exact
}

// BF16 stores truncate, as the reference's store_bfloat does (GEMMHeaders.swift:405-419);
// FP16 stores round to nearest even (a plain MSL half conversion).
__device__ __forceinline__ void store_elem(void *p, size_t i, int prec, float v) {
  if (prec == FP32) {
    reinterpret_cast<float *>(p)[i] = v;
  } else if (prec == FP16) {
    reinterpret_cast<uint16_t *>(p)[i] = __half_as_ushort(__float2half_rn(v));
  } else {
    reinterpret_cast<uint16_t *>(p)[i] = static_cast<uint16_t>(__float_as_uint(v) >> 16);
  }
}

// element (s, d) of a matrix operand: [seq][D] or, transposed, [D][seq]
// (AttentionKernel.swift:189-195: leading dimension = D, or the sequence length when transposed)
__device__ __forceinline__ size_t elem_index(const Operand &op, uint32_t s, uint32_t d) {
  return op.transposed ? static_cast<size_t>(d) * op.seq + s : static_cast<size_t>(s) * op.D + d;
}

// Stage the tile {rows s0..s0+63} x {cols d0..d0+COLS-1} into dst[64][LD] as FP32, zero padded
// (the analogue of the reference's zero-padding async copies, GEMMHeaders.swift:111-114).
template <int COLS, int LD>
__device__ __forceinline__ void load_tile(float *dst, const Operand &op, uint32_t s0, uint32_t d0, uint32_t dEnd,
                                          int tid) {
  constexpr int kElems = kBlock * COLS;
  if (!op.transposed) {
#pragma unroll 4
    for (int e = tid; e < kElems; e += kThreads) {
      int s = e / COLS, d = e % COLS;  // consecutive threads -> consecutive d (coalesced)
      uint32_t gs = s0 + s, gd = d0 + d;
      float v = 0.f;
      if (gs < op.seq && gd < dEnd) v = load_elem(op.ptr, elem_index(op, gs, gd), op.prec);
      dst[s * LD + d] = v;
    }
  } else {
#pragma unroll 4
    for (int e = tid; e < kElems; e += kThreads) {
      int d = e / kBlock, s = e % kBlock;  // consecutive threads -> consecutive s (coalesced)
      uint32_t gs = s0 + s, gd = d0 + d;
      float v = 0.f;
      if (gs < op.seq && gd < dEnd) v = load_elem(op.ptr, elem_index(op, gs, gd), op.prec);
      dst[s * LD + d] = v;
    }
  }
}

// acc[i][j] += sum_d A[a0 + ty + 16 i][d] * B[b0 + tx + 16 j][d]       ("outer product" GEMM,
// AttentionKernel+OuterProduct.swift:18-487: C[par x trav] = A[par x D] . B^T[trav x D])
__device__ __forceinline__ void gemm_nt(float (&acc)[4][4], const Operand &A, uint32_t a0, const Operand &B,
                                        uint32_t b0, float *sA, float *sB, int tid, int tx, int ty) {
  const uint32_t D = A.D;
  for (uint32_t d0 = 0; d0 < D; d0 += kDC) {
    load_tile<kDC, kLDA>(sA, A, a0, d0, D, tid);
    load_tile<kDC, kLDA>(sB, B, b0, d0, D, tid);
    __syncthreads();
#pragma unroll
    for (int d = 0; d < kDC; d += 4) {
      float4 a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4 *>(&sA[(ty + 16 * i) * kLDA + d]);
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = *reinterpret_cast<const float4 *>(&sB[(tx + 16 * j) * kLDA + d]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float s = acc[i][j];
          s = fmaf(a[i].x, b[j].x, s);
          s = fmaf(a[i].y, b[j].y, s);
          s = fmaf(a[i].z, b[j].z, s);
          s = fmaf(a[i].w, b[j].w, s);
          acc[i][j] = s;
        }
    }
    __syncthreads();
  }
}

// acc[q][i][0..3] += sum_k sP[ty + 16 i][k] * X[x0 + k][dlo + 64 q + 4 tx + (0..3)]   ("accumulate"
// GEMM, AttentionKernel+Accumulate.swift:24-582: C[par x D] += A[par x trav] . B[trav x D])
template <int NCH>
__device__ __forceinline__ void accumulate(float (&acc)[NCH][4][4], const float *sP, const Operand &X, uint32_t x0,
                                           uint32_t dlo, uint32_t dhi, float *sX, int tid, int tx, int ty) {
#pragma unroll
  for (int q = 0; q < NCH; ++q) {
    uint32_t d0 = dlo + q * kBlock;
    if (d0 < dhi) {  // uniform across the CTA
      load_tile<kBlock, kLDP>(sX, X, x0, d0, dhi, tid);
      __syncthreads();
#pragma unroll 4
      for (int k = 0; k < kBlock; k += 4) {
        float4 pr[4], xv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) pr[i] = *reinterpret_cast<const float4 *>(&sP[(ty + 16 * i) * kLDP + k]);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) xv[kk] = *reinterpret_cast<const float4 *>(&sX[(k + kk) * kLDP + 4 * tx]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float pk[4] = {pr[i].x, pr[i].y, pr[i].z, pr[i].w};
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            acc[q][i][0] = fmaf(pk[kk], xv[kk].x, acc[q][i][0]);
            acc[q][i][1] = fmaf(pk[kk], xv[kk].y, acc[q][i][1]);
            acc[q][i][2] = fmaf(pk[kk], xv[kk].z, acc[q][i][2]);
            acc[q][i][3] = fmaf(pk[kk], xv[kk].w, acc[q][i][3]);
          }
        }
      }
      __syncthreads();
    }
  }
}

// reduce over the 16 lanes (tx) that share an attention-matrix row
__device__ __forceinline__ float row_max16(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
  return v;
}
__device__ __forceinline__ float row_sum16(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  return v;
}

__device__ __forceinline__ Operand make_operand(const AttentionParams &p, int slot, uint32_t seq, uint32_t b) {
  Operand op;
  size_t bytes = static_cast<size_t>(seq) * p.D * (p.prec[slot] == FP32 ? 4 : 2);
  op.ptr = static_cast<const char *>(p.buf[slot]) + static_cast<size_t>(b) * bytes;
  op.seq = seq;
  op.D = p.D;
  op.prec = p.prec[slot];
  op.transposed = p.transposed[slot];
  return op;
}

// store a [64 x (NCH*64)] register accumulator block to a matrix operand (FP32/FP16/BF16, maybe transposed)
template <int NCH>
__device__ __forceinline__ void store_acc(const float (&acc)[NCH][4][4], const float (&rowScale)[4],
                                          const AttentionParams &p, int slot, uint32_t seq, uint32_t b, uint32_t s0,
                                          uint32_t dlo, uint32_t dhi, int tx, int ty) {
  Operand op = make_operand(p, slot, seq, b);
  void *dst = const_cast<void *>(op.ptr);
#pragma unroll
  for (int q = 0; q < NCH; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t s = s0 + ty + 16 * i;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        uint32_t d = dlo + q * kBlock + 4 * tx + jj;
        if (s < seq && d < dhi) store_elem(dst, elem_index(op, s, d), op.prec, acc[q][i][jj] * rowScale[i]);
      }
    }
}

// ------------------------------------------------------------------------------------------------
// forward: O = softmax(Q K^T / sqrt(D)) V,  L = log2(e) * logsumexp          (one CTA per 64 rows)
// ------------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_forward_kernel(const AttentionParams p) {
  extern __shared__ __align__(16) float smem[];
  float *sA = smem, *sB = sA + kBlock * kLDA, *sP = sB + kBlock * kLDA, *sX = sP + kBlock * kLDP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint32_t b = blockIdx.y, r0 = blockIdx.x * kBlock;

  const Operand Q = make_operand(p, sQ, p.R, b), K = make_operand(p, sK, p.C, b), V = make_operand(p, sV, p.C, b);

  // m = -FLT_MAX, l = denorm_min  (AttentionKernel+Caching.swift:310-311)
  float m[4], l[4];
  float acc[NCH][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = -FLT_MAX;
    l[i] = FLT_TRUE_MIN;
  }
#pragma unroll
  for (int q = 0; q < NCH; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) acc[q][i][jj] = 0.f;

  for (uint32_t c0 = 0; c0 < p.C; c0 += kBlock) {
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
    gemm_nt(s, Q, r0, K, c0, sA, sB, tid, tx, ty);

#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // edge mask (AttentionKernel+Softmax.swift:228-260), then online max / correction / sum (:267-324)
      float mx = -FLT_MAX;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (c0 + tx + 16 * j >= p.C) s[i][j] = -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
      mx = row_max16(mx);
      float m_new = fmaxf(m[i], mx * p.scale_log2);
      float correction = exp2f(m[i] - m_new);
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float pv = exp2f(fmaf(s[i][j], p.scale_log2, -m_new));
        sum += pv;
        sP[(ty + 16 * i) * kLDP + tx + 16 * j] = pv;
      }
      sum = row_sum16(sum);
      l[i] = fmaf(l[i], correction, sum);
      m[i] = m_new;
#pragma unroll
      for (int q = 0; q < NCH; ++q)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) acc[q][i][jj] *= correction;
    }
    // (the __syncthreads inside accumulate() orders the sP writes before its reads)
    accumulate<NCH>(acc, sP, V, c0, 0, p.D, sX, tid, tx, ty);
  }

  // O *= 1/l on the last iteration (AttentionKernel+Source.swift:169-171); L = m + log2(l) (+Caching.swift:373-377)
  float inv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) inv[i] = 1.0f / l[i];
  store_acc<NCH>(acc, inv, p, sO, p.R, b, r0, 0, p.D, tx, ty);
  if (tx == 0 && p.buf[sL] != nullptr) {
    char *Lbase = static_cast<char *>(p.buf[sL]) + static_cast<size_t>(b) * p.R * (p.prec[sL] == FP32 ? 4 : 2);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t r = r0 + ty + 16 * i;
      if (r < p.R) store_elem(Lbase, r, p.prec[sL], m[i] + log2f(l[i]));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward dQ: D = rowsum(dO * O)/sqrt(D);  dQ = sum_c P (dP/sqrt(D) - D) K     (one CTA per 64 rows)
// ------------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_backward_query_kernel(const AttentionParams p) {
  extern __shared__ __align__(16) float smem[];
  float *sA = smem, *sB = sA + kBlock * kLDA, *sP = sB + kBlock * kLDA, *sX = sP + kBlock * kLDP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint32_t b = blockIdx.y, r0 = blockIdx.x * kBlock;

  const Operand Q = make_operand(p, sQ, p.R, b), K = make_operand(p, sK, p.C, b), V = make_operand(p, sV, p.C, b);
  const Operand O = make_operand(p, sO, p.R, b), dO = make_operand(p, sdO, p.R, b);
  const char *Lbase = static_cast<const char *>(p.buf[sL]) + static_cast<size_t>(b) * p.R * (p.prec[sL] == FP32 ? 4 : 2);
  char *Dbase = static_cast<char *>(p.buf[sD]) + static_cast<size_t>(b) * p.R * (p.prec[sD] == FP32 ? 4 : 2);

  // computeD (AttentionKernel+Softmax.swift:32-221): D = (sum_d dO * O) * 1/sqrt(D), kept in FP32
  // registers for this kernel and stored (possibly as BF16) for the dK/dV kernel.
  float Lrow[4], Drow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t r = min(r0 + ty + 16 * i, p.R - 1);  // clamped like clampedParallelizationThreadOffset
    float part = 0.f;
    for (uint32_t d = tx; d < p.D; d += 16)
      part = fmaf(load_elem(dO.ptr, elem_index(dO, r, d), dO.prec), load_elem(O.ptr, elem_index(O, r, d), O.prec), part);
    Drow[i] = row_sum16(part) * p.scale;
    Lrow[i] = load_elem(Lbase, r, p.prec[sL]);
    if (tx == 0 && r0 + ty + 16 * i < p.R) store_elem(Dbase, r, p.prec[sD], Drow[i]);
  }

  float acc[NCH][4][4];
#pragma unroll
  for (int q = 0; q < NCH; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) acc[q][i][jj] = 0.f;

  for (uint32_t c0 = 0; c0 < p.C; c0 += kBlock) {
    float s[4][4], dp[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
    gemm_nt(s, Q, r0, K, c0, sA, sB, tid, tx, ty);    // S  = Q K^T
    gemm_nt(dp, dO, r0, V, c0, sA, sB, tid, tx, ty);  // dP = dO V^T
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // P = exp2(S * log2e/sqrt(D) - L);  dS = P * (dP/sqrt(D) - D)   (+Softmax.swift:419-427)
        float pv = (c0 + tx + 16 * j < p.C) ? exp2f(fmaf(s[i][j], p.scale_log2, -Lrow[i])) : 0.f;
        sP[(ty + 16 * i) * kLDP + tx + 16 * j] = pv * fmaf(dp[i][j], p.scale, -Drow[i]);
      }
    accumulate<NCH>(acc, sP, K, c0, 0, p.D, sX, tid, tx, ty);  // dQ += dS K
  }
  const float one[4] = {1.f, 1.f, 1.f, 1.f};
  store_acc<NCH>(acc, one, p, sdQ, p.R, b, r0, 0, p.D, tx, ty);
}

// ------------------------------------------------------------------------------------------------
// backward dK/dV: dV = sum_r P^T dO;  dK = sum_r dS^T Q      (one CTA per 64 columns x D-slice)
// ------------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_backward_key_value_kernel(const AttentionParams p,
                                                                               uint32_t dSlices) {
  extern __shared__ __align__(16) float smem[];
  float *sA = smem, *sB = sA + kBlock * kLDA, *sPT = sB + kBlock * kLDA, *sX = sPT + kBlock * kLDP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint32_t b = blockIdx.y / dSlices, slice = blockIdx.y % dSlices, c0 = blockIdx.x * kBlock;
  const uint32_t dlo = slice * (NCH * kBlock);
  const uint32_t dhi = min(p.D, dlo + NCH * kBlock);

  const Operand Q = make_operand(p, sQ, p.R, b), K = make_operand(p, sK, p.C, b), V = make_operand(p, sV, p.C, b);
  const Operand dO = make_operand(p, sdO, p.R, b);
  const char *Lbase = static_cast<const char *>(p.buf[sL]) + static_cast<size_t>(b) * p.R * (p.prec[sL] == FP32 ? 4 : 2);
  const char *Dbase = static_cast<const char *>(p.buf[sD]) + static_cast<size_t>(b) * p.R * (p.prec[sD] == FP32 ? 4 : 2);

  float accV[NCH][4][4], accK[NCH][4][4];
#pragma unroll
  for (int q = 0; q < NCH; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) accV[q][i][jj] = accK[q][i][jj] = 0.f;

  for (uint32_t r0 = 0; r0 < p.R; r0 += kBlock) {
    float s[4][4], dp[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
    gemm_nt(s, Q, r0, K, c0, sA, sB, tid, tx, ty);    // S[r][c]
    gemm_nt(dp, dO, r0, V, c0, sA, sB, tid, tx, ty);  // dP[r][c]

    float pv[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t r = r0 + ty + 16 * i;
      uint32_t rc = min(r, p.R - 1);
      // L and D are read back in their memory precision (+Softmax.swift:356-404, 453-468)
      float Lr = load_elem(Lbase, rc, p.prec[sL]);
      float Dr = load_elem(Dbase, rc, p.prec[sD]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float e = (r < p.R) ? exp2f(fmaf(s[i][j], p.scale_log2, -Lr)) : 0.f;
        pv[i][j] = e;
        dp[i][j] = e * fmaf(dp[i][j], p.scale, -Dr);  // dS
        sPT[(tx + 16 * j) * kLDP + ty + 16 * i] = e;  // P^T
      }
    }
    accumulate<NCH>(accV, sPT, dO, r0, dlo, dhi, sX, tid, tx, ty);  // dV += P^T dO
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) sPT[(tx + 16 * j) * kLDP + ty + 16 * i] = dp[i][j];  // dS^T
    accumulate<NCH>(accK, sPT, Q, r0, dlo, dhi, sX, tid, tx, ty);  // dK += dS^T Q
  }
  const float one[4] = {1.f, 1.f, 1.f, 1.f};
  store_acc<NCH>(accV, one, p, sdV, p.C, b, c0, dlo, dhi, tx, ty);
  store_acc<NCH>(accK, one, p, sdK, p.C, b, c0, dlo, dhi, tx, ty);
}

template <typename KernelT>
cudaError_t prepare(KernelT kernel) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
}

inline int chunks_for(uint32_t D) { return (D + kBlock - 1) / kBlock; }

}  // namespace simt

#define MFA_SIMT_DISPATCH(NCHUNKS, KERNEL, GRID, ...)                                     \
  do {                                                                                    \
    cudaError_t e_;                                                                       \
    if ((NCHUNKS) <= 1) {                                                                 \
      e_ = simt::prepare(simt::KERNEL<1>);                                                \
      if (e_ != cudaSuccess) return e_;                                                   \
      simt::KERNEL<1><<<GRID, simt::kThreads, simt::kSmemBytes, stream>>>(__VA_ARGS__);   \
    } else if ((NCHUNKS) <= 2) {                                                          \
      e_ = simt::prepare(simt::KERNEL<2>);                                                \
      if (e_ != cudaSuccess) return e_;                                                   \
      simt::KERNEL<2><<<GRID, simt::kThreads, simt::kSmemBytes, stream>>>(__VA_ARGS__);   \
    } else if ((NCHUNKS) <= 4) {                                                          \
      e_ = simt::prepare(simt::KERNEL<4>);                                                \
      if (e_ != cudaSuccess) return e_;                                                   \
      simt::KERNEL<4><<<GRID, simt::kThreads, simt::kSmemBytes, stream>>>(__VA_ARGS__);   \
    } else {                                                                              \
      e_ = simt::prepare(simt::KERNEL<8>);                                                \
      if (e_ != cudaSuccess) return e_;                                                   \
      simt::KERNEL<8><<<GRID, simt::kThreads, simt::kSmemBytes, stream>>>(__VA_ARGS__);   \
    }                                                                                     \
  } while (0)

cudaError_t launch_simt_forward(const AttentionParams &p, cudaStream_t stream) {
  dim3 grid((p.R + simt::kBlock - 1) / simt::kBlock, p.batch);
  MFA_SIMT_DISPATCH(simt::chunks_for(p.D), simt_forward_kernel, grid, p);
  return cudaGetLastError();
}

cudaError_t launch_simt_backward_query(const AttentionParams &p, cudaStream_t stream) {
  dim3 grid((p.R + simt::kBlock - 1) / simt::kBlock, p.batch);
  MFA_SIMT_DISPATCH(simt::chunks_for(p.D), simt_backward_query_kernel, grid, p);
  return cudaGetLastError();
}

cudaError_t launch_simt_backward_key_value(const AttentionParams &p, cudaStream_t stream) {
  // two accumulators (dV, dK) per thread: keep at most 4 chunks (256 columns) of each in registers and
  // slice larger head dimensions over blockIdx.y (each slice recomputes S and dP).
  int chunks = simt::chunks_for(p.D);
  int nch = chunks <= 1 ? 1 : chunks <= 2 ? 2 : 4;
  uint32_t dSlices = (chunks + nch - 1) / nch;
  dim3 grid((p.C + simt::kBlock - 1) / simt::kBlock, p.batch * dSlices);
  cudaError_t e;
  if (nch == 1) {
    if ((e = simt::prepare(simt::simt_backward_key_value_kernel<1>)) != cudaSuccess) return e;
    simt::simt_backward_key_value_kernel<1><<<grid, simt::kThreads, simt::kSmemBytes, stream>>>(p, dSlices);
  } else if (nch == 2) {
    if ((e = simt::prepare(simt::simt_backward_key_value_kernel<2>)) != cudaSuccess) return e;
    simt::simt_backward_key_value_kernel<2><<<grid, simt::kThreads, simt::kSmemBytes, stream>>>(p, dSlices);
  } else {
    if ((e = simt::prepare(simt::simt_backward_key_value_kernel<4>)) != cudaSuccess) return e;
    simt::simt_backward_key_value_kernel<4><<<grid, simt::kThreads, simt::kSmemBytes, stream>>>(p, dSlices);
  }
  return cudaGetLastError();
}

// Launch geometry reported through AttentionKernel.threadgroupSize / threadgroupMemoryAllocation /
// blockDimensions for this family (AttentionKernel.swift:22-25, 268-270).
void simt_geometry(int /*type*/, uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par, uint32_t *trav,
                   uint32_t *head) {
  *threads = simt::kThreads;
  *smem_bytes = simt::kSmemBytes;
  *par = simt::kBlock;
  *trav = simt::kBlock;
  uint32_t padded = (D + 7) / 8 * 8;  // head block <= pad8(D), AttentionDescriptor.swift:41-54
  *head = padded < (uint32_t)simt::kDC ? padded : simt::kDC;
}

}  // namespace mfa
