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
// One body per kernel type (forward_body, backward_query_body, backward_key_value_body) serves every call form: the
// call's layout (fixed-length, packed sequences, a paged K/V cache) and its mask (causal or none, or a sliding window)
// are template parameters, and each __global__ entry point fixes both.
// Causal (p.causal): row r sees column c iff c <= r + offset (C - R, or Cs - Rs of a sequence); the loops skip the
// 64-blocks no row of the CTA can see, the mask is applied with the edge mask, and a row that sees no column gets
// O = 0, L = +inf.
// Grouped K/V (p.group query problems per K/V problem): query problem b reads K / V problem b / p.group, and a dK/dV
// CTA sums over the rows of every query problem of its group.
// Sliding window (Band, the simt_band_* kernels): row r sees column c iff r + offset - left <= c <= r + offset + right;
// the loops visit only the 64-blocks that meet the CTA's band.
//
// Tiling: one CTA = 256 threads = a 64 x 64 block of the attention matrix; thread (tx, ty) owns
// the 4 x 4 patch {rows ty+16i} x {cols tx+16j}.  Operands are staged through shared memory as
// FP32 in 64 x 32 (contraction over D) and 64 x 64 (accumulation) tiles; output accumulators
// (64 x D) live in registers, 4 rows x (D/16) columns per thread.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include <type_traits>

#include "attention_params.h"
#include "device_state.h"
#include "mfa_b200.h"

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

// Paged K/V (the paged forward): the keys of one sequence and K/V head in a pool [pages][P][kv_heads][D], row-major;
// key s is pool row paged_row(s), and keys at or past seq read as zero.  Under a window (kBand) keys below `first`
// read as zero too, without touching their page-table entries or pages (DESIGN "Paged page skipping").
template <bool kBand>
struct PagedOperand {
  const void *ptr;
  const int32_t *table;  // the sequence's page_table row
  PagedKV pk;            // pages, page_shift, kv_heads
  uint32_t seq;          // Cs, or under a window the end of the keys the tile's band meets
  uint32_t D, head;
  int prec;
};
template <>
struct PagedOperand<true> : PagedOperand<false> {
  uint32_t first;
};

template <int COLS, int LD, bool kBand>
__device__ __forceinline__ void load_tile(float *dst, const PagedOperand<kBand> &op, uint32_t s0, uint32_t d0,
                                          uint32_t dEnd, int tid) {
  constexpr int kElems = kBlock * COLS;
#pragma unroll 4
  for (int e = tid; e < kElems; e += kThreads) {
    const int s = e / COLS, d = e % COLS;
    const uint32_t gs = s0 + s, gd = d0 + d;
    bool read = gs < op.seq && gd < dEnd;
    if constexpr (kBand) read = read && gs >= op.first;
    float v = 0.f;
    if (read) {
      const size_t row = paged_row(op.pk, op.table, gs);
      v = load_elem(op.ptr, (row * op.pk.kv_heads + op.head) * op.D + gd, op.prec);
    }
    dst[s * LD + d] = v;
  }
}

// acc[i][j] += sum_d A[a0 + ty + 16 i][d] * B[b0 + tx + 16 j][d]       ("outer product" GEMM,
// AttentionKernel+OuterProduct.swift:18-487: C[par x trav] = A[par x D] . B^T[trav x D])
template <class OperandB>
__device__ __forceinline__ void gemm_nt(float (&acc)[4][4], const Operand &A, uint32_t a0, const OperandB &B,
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
template <int NCH, class OperandX>
__device__ __forceinline__ void accumulate(float (&acc)[NCH][4][4], const float *sP, const OperandX &X, uint32_t x0,
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

// the R statistics (L or D) of problem b in `slot`
__device__ __forceinline__ char *stat_row(const AttentionParams &p, int slot, uint32_t b) {
  return static_cast<char *>(p.buf[slot]) + static_cast<size_t>(b) * p.R * (p.prec[slot] == FP32 ? 4 : 2);
}

// ------------------------------------------------------------------------------------------------
// Call forms (Layout).  A CTA works on a span: the whole R x C problem (kFixed, with the causal offset C - R that
// p.causal_offset holds), or sequence blockIdx.z of a packed (kPacked) or paged (kPaged) call, with its offset Cs - Rs.
// Rows past a span's end read as zeros (Operand::seq).  A fixed span starts at row 0 and covers the whole operand, so
// transposed fixed-length operands keep their leading dimension; packed operands are row-major (a transposed operand's
// leading dimension is the whole buffer, which Operand does not carry; kernel.cpp rejects them).
// ------------------------------------------------------------------------------------------------
enum class Layout { kFixed, kPacked, kPaged };

struct Span {
  SequenceSpan s;
  int offset;  // row r's diagonal is column r + offset
};
template <Layout kLayout>
__device__ __forceinline__ Span span_of(const AttentionParams &p, const Sequences &seq, const PagedKV &pk) {
  Span sp;
  if constexpr (kLayout == Layout::kFixed) {
    sp.s = SequenceSpan{0, p.R, 0, p.C};
    sp.offset = p.causal_offset;
  } else {
    if constexpr (kLayout == Layout::kPacked) {
      sp.s = sequence_span(seq, blockIdx.z);
    } else {
      sp.s = paged_span(pk, blockIdx.z);
    }
    sp.offset = static_cast<int>(sp.s.C) - static_cast<int>(sp.s.R);
  }
  return sp;
}
// rows [first, first + len) of problem b of `slot`, whose buffer holds `rows` rows per problem
__device__ __forceinline__ Operand span_operand(const AttentionParams &p, int slot, uint32_t rows, uint32_t b,
                                                uint32_t first, uint32_t len) {
  Operand op = make_operand(p, slot, rows, b);
  op.ptr = static_cast<const char *>(op.ptr) + static_cast<size_t>(first) * p.D * (p.prec[slot] == FP32 ? 4 : 2);
  op.seq = len;
  return op;
}
__device__ __forceinline__ Operand span_query(const AttentionParams &p, int slot, uint32_t b, const Span &sp) {
  return span_operand(p, slot, p.R, b, sp.s.q0, sp.s.R);
}
__device__ __forceinline__ Operand span_key(const AttentionParams &p, int slot, uint32_t kv, const Span &sp) {
  return span_operand(p, slot, p.C, kv, sp.s.k0, sp.s.C);
}
__device__ __forceinline__ char *span_stats(const AttentionParams &p, int slot, uint32_t b, const Span &sp) {
  return stat_row(p, slot, b) + static_cast<size_t>(sp.s.q0) * (p.prec[slot] == FP32 ? 4 : 2);
}
// store a [64 x (NCH*64)] register accumulator block, each row scaled, to the rows [0, op.seq) of `op`
template <int NCH>
__device__ __forceinline__ void span_store(const float (&acc)[NCH][4][4], const float (&rowScale)[4], const Operand &op,
                                           uint32_t s0, uint32_t dlo, uint32_t dhi, int tx, int ty) {
  void *dst = const_cast<void *>(op.ptr);
#pragma unroll
  for (int q = 0; q < NCH; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t s = s0 + ty + 16 * i;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const uint32_t d = dlo + q * kBlock + 4 * tx + jj;
        if (s < op.seq && d < dhi) store_elem(dst, elem_index(op, s, d), op.prec, acc[q][i][jj] * rowScale[i]);
      }
    }
}
template <int NCH>
__device__ __forceinline__ void zero_acc(float (&acc)[NCH][4][4]) {
#pragma unroll
  for (int q = 0; q < NCH; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) acc[q][i][jj] = 0.f;
}

// ------------------------------------------------------------------------------------------------
// Masks, a compile-time choice.  kBand = false: the edge, and with p.causal the causal mask (row r sees column c iff
// c <= r + offset).  kBand = true: the edge and a sliding window (row r sees column c iff r + offset - left <= c <=
// r + offset + right; the host passes a causal window as right = 0), in 64-bit arithmetic since a side may be as large
// as INT32_MAX.  They stay apart so that the kernels without a window, the family's main path, do no 64-bit work.
// ------------------------------------------------------------------------------------------------
// The columns [*first, *end) of the 64-blocks that the rows [r0, min(r0 + 64, Rs)) see, *first rounded down to a block
template <bool kBand>
__device__ __forceinline__ void key_blocks(const AttentionParams &p, const Span &sp, const Band &band, uint32_t r0,
                                           uint32_t *first, uint32_t *end) {
  if constexpr (kBand) {
    const int64_t lo = static_cast<int64_t>(r0) + sp.offset - band.left;
    const int64_t hi = static_cast<int64_t>(min(r0 + kBlock, sp.s.R)) - 1 + sp.offset + band.right;
    *first = lo <= 0 ? 0u : static_cast<uint32_t>(min(lo, static_cast<int64_t>(sp.s.C))) / kBlock * kBlock;
    *end = hi < 0 ? 0u : static_cast<uint32_t>(min(hi + 1, static_cast<int64_t>(sp.s.C)));
  } else {
    *first = 0;
    if (!p.causal) {
      *end = sp.s.C;
    } else {
      const int last = static_cast<int>(min(r0 + kBlock, sp.s.R)) - 1 + sp.offset;  // last column of the last row
      *end = last < 0 ? 0u : min(sp.s.C, static_cast<uint32_t>(last) + 1);
    }
  }
}
// The rows [*first, *end) of the 64-blocks that see the columns [c0, min(c0 + 64, Cs)), *first rounded down to a block
template <bool kBand>
__device__ __forceinline__ void query_blocks(const AttentionParams &p, const Span &sp, const Band &band, uint32_t c0,
                                             uint32_t *first, uint32_t *end) {
  if constexpr (kBand) {
    const int64_t lo = static_cast<int64_t>(c0) - sp.offset - band.right;
    const int64_t hi = static_cast<int64_t>(min(c0 + kBlock, sp.s.C)) - 1 - sp.offset + band.left;
    *first = lo <= 0 ? 0u : static_cast<uint32_t>(min(lo, static_cast<int64_t>(sp.s.R))) / kBlock * kBlock;
    *end = hi < 0 ? 0u : static_cast<uint32_t>(min(hi + 1, static_cast<int64_t>(sp.s.R)));
  } else {
    const int lo = static_cast<int>(c0) - sp.offset;  // the first row that sees column c0
    *first = p.causal && lo > 0 ? static_cast<uint32_t>(lo) / kBlock * kBlock : 0;
    *end = sp.s.R;
  }
}
// column c is past the edge (tested with kEdge), or hidden from row r
template <bool kBand, bool kEdge = true>
__device__ __forceinline__ bool masked(const AttentionParams &p, const Span &sp, const Band &band, uint32_t r,
                                       uint32_t c) {
  if constexpr (kBand) {
    const int64_t d = static_cast<int64_t>(c) - r - sp.offset;  // column - (row + offset)
    return (kEdge && c >= sp.s.C) || d > band.right || -d > band.left;
  } else {
    return (kEdge && c >= sp.s.C) || (p.causal && static_cast<int>(c) > static_cast<int>(r) + sp.offset);
  }
}
// row r sees no column: the span has no keys, or the row's diagonal (band) lies wholly before or past them
template <bool kBand>
__device__ __forceinline__ bool row_empty(const AttentionParams &p, const Span &sp, const Band &band, uint32_t r) {
  if constexpr (kBand) {
    const int64_t diag = static_cast<int64_t>(r) + sp.offset;
    return sp.s.C == 0 || diag + band.right < 0 || diag - band.left >= static_cast<int64_t>(sp.s.C);
  } else {
    return sp.s.C == 0 || (p.causal && static_cast<int>(r) + sp.offset < 0);
  }
}

// K or V (`slot`) of K/V head kv for the forward tile of rows [r0, r0 + 64): the span's rows of the operand, or a paged
// call's keys through its page table.  Under a window, a paged operand reads only the keys the tile's band can meet:
// none before the band of its first row, nor any from the end of its key blocks on.
template <Layout kLayout, bool kBand>
__device__ __forceinline__ auto key_operand(const AttentionParams &p, int slot, uint32_t kv, const Span &sp,
                                            const PagedKV &pk, const Band &band, uint32_t r0) {
  if constexpr (kLayout == Layout::kPaged) {
    PagedOperand<kBand> op;
    op.ptr = p.buf[slot];
    op.table = pk.page_table + static_cast<size_t>(blockIdx.z) * pk.page_stride;
    op.pk = pk;
    op.seq = sp.s.C;
    op.D = p.D;
    op.head = kv;
    op.prec = p.prec[slot];
    if constexpr (kBand) {
      uint32_t c_first;
      key_blocks<true>(p, sp, band, r0, &c_first, &op.seq);
      op.first =
          static_cast<uint32_t>(max(static_cast<int64_t>(r0) + sp.offset - band.left, static_cast<int64_t>(0)));
    }
    return op;
  } else {
    return span_key(p, slot, kv, sp);
  }
}

// ------------------------------------------------------------------------------------------------
// forward: O = softmax(Q K^T / sqrt(D)) V,  L = log2(e) * logsumexp          (one CTA per 64 rows)
// ------------------------------------------------------------------------------------------------
template <int NCH, Layout kLayout, bool kBand>
__device__ __forceinline__ void forward_body(const AttentionParams &p, const Sequences &seq, const PagedKV &pk,
                                             const Band &band) {
  extern __shared__ __align__(16) float smem[];
  float *sA = smem, *sB = sA + kBlock * kLDA, *sP = sB + kBlock * kLDA, *sX = sP + kBlock * kLDP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint32_t b = blockIdx.y, r0 = blockIdx.x * kBlock;
  const Span sp = span_of<kLayout>(p, seq, pk);
  if (kLayout != Layout::kFixed && r0 >= sp.s.R) return;  // a tile past the sequence's end (a fixed grid has none)
  const Operand Q = span_query(p, sQ, b, sp);
  const auto K = key_operand<kLayout, kBand>(p, sK, b / p.group, sp, pk, band, r0),
             V = key_operand<kLayout, kBand>(p, sV, b / p.group, sp, pk, band, r0);

  // m = -FLT_MAX, l = denorm_min  (AttentionKernel+Caching.swift:310-311)
  float m[4], l[4], acc[NCH][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = -FLT_MAX;
    l[i] = FLT_TRUE_MIN;
  }
  zero_acc(acc);
  uint32_t c_first, c_end;
  key_blocks<kBand>(p, sp, band, r0, &c_first, &c_end);
  for (uint32_t c0 = c_first; c0 < c_end; c0 += kBlock) {
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
    gemm_nt(s, Q, r0, K, c0, sA, sB, tid, tx, ty);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // mask (AttentionKernel+Softmax.swift:228-260), then online max / correction / sum (:267-324)
      float mx = -FLT_MAX;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (masked<kBand>(p, sp, band, r0 + ty + 16 * i, c0 + tx + 16 * j)) s[i][j] = -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
      mx = row_max16(mx);
      const float m_new = fmaxf(m[i], mx * p.scale_log2), correction = exp2f(m[i] - m_new);
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float pv = exp2f(fmaf(s[i][j], p.scale_log2, -m_new));
        sum += pv;
        sP[(ty + 16 * i) * kLDP + tx + 16 * j] = pv;
      }
      l[i] = fmaf(l[i], correction, row_sum16(sum));
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
  // a row that sees no column gets O = 0 and L = +inf
  float inv[4];
  bool empty[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    empty[i] = row_empty<kBand>(p, sp, band, r0 + ty + 16 * i);
    inv[i] = empty[i] ? 0.f : 1.0f / l[i];
  }
  span_store<NCH>(acc, inv, span_query(p, sO, b, sp), r0, 0, p.D, tx, ty);
  if (tx == 0 && p.buf[sL] != nullptr) {
    char *Lbase = span_stats(p, sL, b, sp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t r = r0 + ty + 16 * i;
      if (r < sp.s.R) store_elem(Lbase, r, p.prec[sL], empty[i] ? INFINITY : m[i] + log2f(l[i]));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward dQ: D = rowsum(dO * O)/sqrt(D);  dQ = sum_c P (dP/sqrt(D) - D) K     (one CTA per 64 rows)
// ------------------------------------------------------------------------------------------------
template <int NCH, Layout kLayout, bool kBand>
__device__ __forceinline__ void backward_query_body(const AttentionParams &p, const Sequences &seq, const Band &band) {
  static_assert(kLayout != Layout::kPaged, "paged calls are forward only");
  extern __shared__ __align__(16) float smem[];
  float *sA = smem, *sB = sA + kBlock * kLDA, *sP = sB + kBlock * kLDA, *sX = sP + kBlock * kLDP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint32_t b = blockIdx.y, r0 = blockIdx.x * kBlock;
  const Span sp = span_of<kLayout>(p, seq, PagedKV{});
  if (kLayout != Layout::kFixed && r0 >= sp.s.R) return;  // a tile past the sequence's end (a fixed grid has none)
  const Operand Q = span_query(p, sQ, b, sp), K = span_key(p, sK, b / p.group, sp), V = span_key(p, sV, b / p.group, sp);
  const Operand O = span_query(p, sO, b, sp), dO = span_query(p, sdO, b, sp);
  const char *Lbase = span_stats(p, sL, b, sp);
  char *Dbase = span_stats(p, sD, b, sp);

  // computeD (AttentionKernel+Softmax.swift:32-221): D = (sum_d dO * O) * 1/sqrt(D), kept in FP32
  // registers for this kernel and stored (possibly as BF16) for the dK/dV kernel.
  float Lrow[4], Drow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t r = min(r0 + ty + 16 * i, sp.s.R - 1);  // clamped like clampedParallelizationThreadOffset
    float part = 0.f;
    for (uint32_t d = tx; d < p.D; d += 16)
      part = fmaf(load_elem(dO.ptr, elem_index(dO, r, d), dO.prec), load_elem(O.ptr, elem_index(O, r, d), O.prec), part);
    Drow[i] = row_sum16(part) * p.scale;
    Lrow[i] = load_elem(Lbase, r, p.prec[sL]);
    if (tx == 0 && r0 + ty + 16 * i < sp.s.R) store_elem(Dbase, r, p.prec[sD], Drow[i]);
  }

  float acc[NCH][4][4];
  zero_acc(acc);
  uint32_t c_first, c_end;
  key_blocks<kBand>(p, sp, band, r0, &c_first, &c_end);
  for (uint32_t c0 = c_first; c0 < c_end; c0 += kBlock) {
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
        const float pv = !masked<kBand>(p, sp, band, r0 + ty + 16 * i, c0 + tx + 16 * j)
                             ? exp2f(fmaf(s[i][j], p.scale_log2, -Lrow[i]))
                             : 0.f;
        sP[(ty + 16 * i) * kLDP + tx + 16 * j] = pv * fmaf(dp[i][j], p.scale, -Drow[i]);
      }
    accumulate<NCH>(acc, sP, K, c0, 0, p.D, sX, tid, tx, ty);  // dQ += dS K
  }
  const float one[4] = {1.f, 1.f, 1.f, 1.f};
  span_store<NCH>(acc, one, span_query(p, sdQ, b, sp), r0, 0, p.D, tx, ty);
}

// ------------------------------------------------------------------------------------------------
// backward dK/dV: dV = sum_r P^T dO;  dK = sum_r dS^T Q      (one CTA per 64 columns x D-slice)
// Grouped K/V: blockIdx.y covers K/V heads, and the sums run over the rows of every query head of the group.
// ------------------------------------------------------------------------------------------------
template <int NCH, Layout kLayout, bool kBand>
__device__ __forceinline__ void backward_key_value_body(const AttentionParams &p, uint32_t dSlices,
                                                        const Sequences &seq, const Band &band) {
  static_assert(kLayout != Layout::kPaged, "paged calls are forward only");
  extern __shared__ __align__(16) float smem[];
  float *sA = smem, *sB = sA + kBlock * kLDA, *sPT = sB + kBlock * kLDA, *sX = sPT + kBlock * kLDP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint32_t kvb = blockIdx.y / dSlices, slice = blockIdx.y % dSlices, c0 = blockIdx.x * kBlock;
  const uint32_t dlo = slice * (NCH * kBlock), dhi = min(p.D, dlo + NCH * kBlock);
  const Span sp = span_of<kLayout>(p, seq, PagedKV{});
  // a tile past the sequence's end (a fixed grid has none); columns that no row sees still store their zeros
  if (kLayout != Layout::kFixed && c0 >= sp.s.C) return;
  const Operand K = span_key(p, sK, kvb, sp), V = span_key(p, sV, kvb, sp);
  float accV[NCH][4][4], accK[NCH][4][4];
  zero_acc(accV);
  zero_acc(accK);
  uint32_t r_first, r_end;
  query_blocks<kBand>(p, sp, band, c0, &r_first, &r_end);
  // Columns past Cs need no mask here: their keys read as zero, and their dK / dV rows are never stored.  The fixed-length
  // kernels leave them unmasked; the packed ones keep the test, without which ptxas spills the packed kernel at NCH = 4.
  constexpr bool kColumnEdge = kLayout != Layout::kFixed;
  for (uint32_t b = kvb * p.group; b < (kvb + 1) * p.group; ++b) {  // the query heads of the group
    const Operand Q = span_query(p, sQ, b, sp), dO = span_query(p, sdO, b, sp);
    const char *Lbase = span_stats(p, sL, b, sp), *Dbase = span_stats(p, sD, b, sp);
    for (uint32_t r0 = r_first; r0 < r_end; r0 += kBlock) {
      float s[4][4], dp[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
      gemm_nt(s, Q, r0, K, c0, sA, sB, tid, tx, ty);    // S[r][c]
      gemm_nt(dp, dO, r0, V, c0, sA, sB, tid, tx, ty);  // dP[r][c]
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t r = r0 + ty + 16 * i, rc = min(r, sp.s.R - 1);
        // L and D are read back in their memory precision (+Softmax.swift:356-404, 453-468)
        const float Lr = load_elem(Lbase, rc, p.prec[sL]), Dr = load_elem(Dbase, rc, p.prec[sD]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float e = r < sp.s.R && !masked<kBand, kColumnEdge>(p, sp, band, r, c0 + tx + 16 * j)
                              ? exp2f(fmaf(s[i][j], p.scale_log2, -Lr))
                              : 0.f;
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
  }
  const float one[4] = {1.f, 1.f, 1.f, 1.f};
  span_store<NCH>(accV, one, span_key(p, sdV, kvb, sp), c0, dlo, dhi, tx, ty);
  span_store<NCH>(accK, one, span_key(p, sdK, kvb, sp), c0, dlo, dhi, tx, ty);
}

// ------------------------------------------------------------------------------------------------
// Entry points: fixed-length, packed (_varlen) and paged (forward only) calls without a window, and the same forms under
// a window (simt_band_*, with Layout a template parameter).  Each is its body with the form fixed at compile time.
// ------------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_forward_kernel(const AttentionParams p) {
  forward_body<NCH, Layout::kFixed, false>(p, Sequences{}, PagedKV{}, Band{});
}
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_forward_kernel_varlen(const AttentionParams p, const Sequences seq) {
  forward_body<NCH, Layout::kPacked, false>(p, seq, PagedKV{}, Band{});
}
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_forward_kernel_paged(const AttentionParams p, const PagedKV pk) {
  forward_body<NCH, Layout::kPaged, false>(p, Sequences{}, pk, Band{});
}
template <int NCH, Layout kLayout>
__global__ void __launch_bounds__(kThreads, 1) simt_band_forward_kernel(const AttentionParams p, const Sequences seq,
                                                                        const PagedKV pk, const Band band) {
  forward_body<NCH, kLayout, true>(p, seq, pk, band);
}

template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_backward_query_kernel(const AttentionParams p) {
  backward_query_body<NCH, Layout::kFixed, false>(p, Sequences{}, Band{});
}
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_backward_query_kernel_varlen(const AttentionParams p,
                                                                                 const Sequences seq) {
  backward_query_body<NCH, Layout::kPacked, false>(p, seq, Band{});
}
template <int NCH, Layout kLayout>
__global__ void __launch_bounds__(kThreads, 1) simt_band_backward_query_kernel(const AttentionParams p,
                                                                               const Sequences seq, const Band band) {
  backward_query_body<NCH, kLayout, true>(p, seq, band);
}

template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_backward_key_value_kernel(const AttentionParams p,
                                                                               uint32_t dSlices) {
  backward_key_value_body<NCH, Layout::kFixed, false>(p, dSlices, Sequences{}, Band{});
}
template <int NCH>
__global__ void __launch_bounds__(kThreads, 1) simt_backward_key_value_kernel_varlen(const AttentionParams p,
                                                                                      uint32_t dSlices,
                                                                                      const Sequences seq) {
  backward_key_value_body<NCH, Layout::kPacked, false>(p, dSlices, seq, Band{});
}
template <int NCH, Layout kLayout>
__global__ void __launch_bounds__(kThreads, 1) simt_band_backward_key_value_kernel(const AttentionParams p,
                                                                                   uint32_t dSlices,
                                                                                   const Sequences seq,
                                                                                   const Band band) {
  backward_key_value_body<NCH, kLayout, true>(p, dSlices, seq, band);
}

inline int chunks_for(uint32_t D) { return (D + kBlock - 1) / kBlock; }

// Calls f(std::integral_constant<int, NCH>()) for the fewest of 1 / 2 / 4 / 8 (at most kMax) column chunks per CTA
// that cover `chunks`
template <int kMax, class F>
cudaError_t with_chunks(int chunks, F f) {
  static_assert(kMax == 4 || kMax == 8, "the kernels are instantiated for 1 / 2 / 4 / 8 chunks");
  if (chunks <= 1) return f(std::integral_constant<int, 1>());
  if (chunks <= 2) return f(std::integral_constant<int, 2>());
  if constexpr (kMax == 4) {
    return f(std::integral_constant<int, 4>());
  } else {
    if (chunks <= 4) return f(std::integral_constant<int, 4>());
    return f(std::integral_constant<int, 8>());
  }
}

// kernel<<<grid>>>(args...) after the opt-in to kSmemBytes of dynamic shared memory (once per kernel and device)
template <typename Kernel, typename... Args>
cudaError_t launch(Kernel kernel, dim3 grid, cudaStream_t stream, const Args &...args) {
  cudaError_t e = ensure_max_dynamic_smem(reinterpret_cast<const void *>(kernel), kSmemBytes, current_device());
  if (e != cudaSuccess) return e;
  kernel<<<grid, kThreads, kSmemBytes, stream>>>(args...);
  return cudaGetLastError();
}

}  // namespace simt

// Packed sequences (seq): the grid's x axis covers the longest sequence and its z axis the sequences (row-major
// operands: kernel.cpp rejects transposed ones)
static dim3 simt_grid(uint32_t rows, uint32_t y, const Sequences *seq) {
  return dim3((rows + simt::kBlock - 1) / simt::kBlock, y, seq ? seq->count : 1);
}

static cudaError_t launch_forward(const AttentionParams &p, const AttentionCall &call, cudaStream_t stream) {
  const Sequences *seq = call.seq;
  const PagedKV *pk = call.pk;
  const Band *band = call.band;
  const uint32_t rows = pk ? pk->max_row : (seq ? seq->max_row : p.R);
  const dim3 grid((rows + simt::kBlock - 1) / simt::kBlock, p.batch, pk ? pk->count : (seq ? seq->count : 1));
  return simt::with_chunks<8>(simt::chunks_for(p.D), [&](auto nch) {
    constexpr int NCH = decltype(nch)::value;
    using simt::Layout;
    if (band && pk)
      return simt::launch(simt::simt_band_forward_kernel<NCH, Layout::kPaged>, grid, stream, p, Sequences{}, *pk, *band);
    if (band && seq)
      return simt::launch(simt::simt_band_forward_kernel<NCH, Layout::kPacked>, grid, stream, p, *seq, PagedKV{}, *band);
    if (band)
      return simt::launch(simt::simt_band_forward_kernel<NCH, Layout::kFixed>, grid, stream, p, Sequences{}, PagedKV{},
                          *band);
    if (pk) return simt::launch(simt::simt_forward_kernel_paged<NCH>, grid, stream, p, *pk);
    if (seq) return simt::launch(simt::simt_forward_kernel_varlen<NCH>, grid, stream, p, *seq);
    return simt::launch(simt::simt_forward_kernel<NCH>, grid, stream, p);
  });
}

static cudaError_t launch_backward_query(const AttentionParams &p, const Sequences *seq, const Band *band,
                                        cudaStream_t stream) {
  const dim3 grid = simt_grid(seq ? seq->max_row : p.R, p.batch, seq);
  return simt::with_chunks<8>(simt::chunks_for(p.D), [&](auto nch) {
    constexpr int NCH = decltype(nch)::value;
    using simt::Layout;
    if (band && seq)
      return simt::launch(simt::simt_band_backward_query_kernel<NCH, Layout::kPacked>, grid, stream, p, *seq, *band);
    if (band)
      return simt::launch(simt::simt_band_backward_query_kernel<NCH, Layout::kFixed>, grid, stream, p, Sequences{},
                          *band);
    if (seq) return simt::launch(simt::simt_backward_query_kernel_varlen<NCH>, grid, stream, p, *seq);
    return simt::launch(simt::simt_backward_query_kernel<NCH>, grid, stream, p);
  });
}

static cudaError_t launch_backward_key_value(const AttentionParams &p, const Sequences *seq, const Band *band,
                                            cudaStream_t stream) {
  // two accumulators (dV, dK) per thread: keep at most 4 chunks (256 columns) of each in registers and
  // slice larger head dimensions over blockIdx.y (each slice recomputes S and dP).
  const int chunks = simt::chunks_for(p.D);
  return simt::with_chunks<4>(chunks, [&](auto nch) {
    constexpr int NCH = decltype(nch)::value;
    const uint32_t dSlices = (chunks + NCH - 1) / NCH;
    // one CTA row per K/V head
    const dim3 grid = simt_grid(seq ? seq->max_column : p.C, p.batch / p.group * dSlices, seq);
    using simt::Layout;
    if (band && seq)
      return simt::launch(simt::simt_band_backward_key_value_kernel<NCH, Layout::kPacked>, grid, stream, p, dSlices,
                          *seq, *band);
    if (band)
      return simt::launch(simt::simt_band_backward_key_value_kernel<NCH, Layout::kFixed>, grid, stream, p, dSlices,
                          Sequences{}, *band);
    if (seq) return simt::launch(simt::simt_backward_key_value_kernel_varlen<NCH>, grid, stream, p, dSlices, *seq);
    return simt::launch(simt::simt_backward_key_value_kernel<NCH>, grid, stream, p, dSlices);
  });
}

cudaError_t launch_simt(int type, const AttentionParams &p, const AttentionCall &call, cudaStream_t stream) {
  switch (type) {
    case MFA_FORWARD: return launch_forward(p, call, stream);
    case MFA_BACKWARD_QUERY: return launch_backward_query(p, call.seq, call.band, stream);
    default: return launch_backward_key_value(p, call.seq, call.band, stream);
  }
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
