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
//
// Causal (kCausal, bottom-right aligned: query row i sees key j iff j <= i + delta, delta = C - R): every CTA visits only
// the traversal blocks its rows can see, and only the blocks that cross the diagonal mask elements (S -> -inf before the
// softmax / before P = exp2(S - L)).  A row that sees no key (i < R - C) gets O = 0, L = +inf, D = 0, dQ = 0.
//
// Grouped K/V (`group` query heads per K/V head, a launch-time value): forward and dQ read K/V head head / group; the
// dK/dV grid's y axis is K/V heads, and a CTA walks the query blocks of every query head of its group, so dK and dV
// are the group sums, accumulated in registers without atomics.
//
// Every forward entry point takes the three tensor maps and one FwdArgs (below), whose fields each form reads as it
// needs; launch_forward picks the entry point of a call's form and fills FwdArgs once.
//
// Packed sequences (the packed_* entry points, kVarlen in the shared bodies): grid.z is the sequence; a CTA takes its
// sequence's rows from the offset tables, leaves when its tile starts past the sequence's end, works on the sequence's
// R, C and delta, and zeroes the rows of its last streamed block that belong to the next sequence.  Unsplit, except in
// the split_forward_* kernels (kSplit): there grid.x is tiles x splits, each CTA walks one ceiling-cut range of its
// tile's visible key blocks, and merge_sequence_splits merges the partials of the sequence's rows.
//
// Paged K/V (the paged_* forward, KVLayout::kPaged in forward_body): queries packed as above, keys and values in pools
// [pages][P][kv_heads][D] read through a 3-D tensor map {D, kv_heads, pool rows} with boxes of 64 x 1 x min(P, BN), so
// each box lands as the same [rows][64] swizzled tile.  A stage takes BN / min(P, BN) boxes per column chunk and tensor,
// each at the pool row of its page; thread 0 reads the block's page ids just before it issues its boxes.
//
// Sliding window (the band_* entry points, kBand in the shared bodies; Band in attention_params.h): row i sees key j iff
// i + delta - left <= j <= i + delta + right, with left and right runtime values, so one instantiation serves every
// window.  A CTA visits only the traversal blocks that meet its rows' (keys') band; only blocks that cross an edge of the
// band are masked (mask_outside_band, whose edges are 64-bit: a side may be as large as INT32_MAX).  The bodies run with kCausal set, which brings the empty-row handling (reference value 0 for a
// row without a key yet, L = -inf split partials, merge_splits<true>).  A fixed-length split range counts from the
// tile's first visible block.  Paged: boxes of pages wholly outside the tile's band are not issued (their page-table
// entries are never read); their bytes are completed on the barrier by hand and their rows zeroed.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "attention_params.h"
#include "backward_common.cuh"
#include "device_state.h"
#include "mfa_b200.h"
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

// The first of the two accumulator rows that thread t of a warpgroup holds (the second is 8 below it; wgmma.cuh)
__device__ __forceinline__ uint32_t frag_row(uint32_t t) { return (t / 32) * 16 + (t % 32) / 4; }

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

// acc = A B^T over the DCH * 64 head columns: A = rows [a0, a0 + 64) of the ROWS_A-row tile at sA, B = the N-row tile
// at sB, both K-major.  Issues the wgmmas only; the caller fences, commits and waits.
template <uint32_t DCH, uint32_t N, bool kBF16, uint32_t ROWS_A>
__device__ __forceinline__ void mma_ss(float (&acc)[N / 2], uint32_t sA, uint32_t a0, uint32_t sB) {
#pragma unroll
  for (uint32_t kk = 0; kk < DCH * 4; ++kk)
    Wgmma<N, kBF16>::ss(acc, desc_kmajor<ROWS_A>(sA, a0, kk), desc_kmajor<N>(sB, 0, kk), kk > 0);
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

// Shared memory of a kernel from its 1024-byte-aligned base: the resident tiles, two ring stages of two streamed tiles
// each, then the barriers.  kSmemBytes adds the slack for aligning the base.
template <uint32_t RESIDENT, uint32_t TILE>
struct SmemLayout {
  static constexpr uint32_t kResidentBytes = RESIDENT, kStageBytes = 2 * TILE;
  static constexpr uint32_t kBarOffset = RESIDENT + 2 * kStageBytes;
  static constexpr uint32_t kSmemBytes = 1024 + kBarOffset + kBarBytes;
};

// The two-stage ring of the streamed tiles.  Traversal step n goes to stage n & 1, which completes on bar[1 + (n & 1)]
// with parity (n >> 1) & 1; bar[0] tracks the resident tiles.  Thread 0 issues every load; a load callback
// load(n, dst, bar) issues the TMA loads of step n's two tiles into dst.  The callbacks are taken by reference: copying
// the closures into these calls made ptxas schedule the dK/dV kernels differently (1-2 registers, more instructions).
//
// kRelease: stages are freed through mbarriers instead of a CTA-wide barrier, so the two warpgroups drift apart and one's
// softmax can run while the other's wgmmas hold the tensor cores.  Each warpgroup arrives on the empty barrier
// bar[3 + s] of a stage it is done with (count 2); thread 0 waits on it before it refills the stage (refill).
template <class Smem, bool kRelease = false>
struct Ring {
  uint8_t *base;
  uint64_t *bar;

  __device__ __forceinline__ explicit Ring(uint8_t *smem)
      : base(align1024(smem)), bar(reinterpret_cast<uint64_t *>(base + Smem::kBarOffset)) {}
  // stage s starts kResidentBytes + s kStageBytes into the base
  __device__ __forceinline__ uint8_t *stage(uint32_t n) const {
    return base + Smem::kResidentBytes + (n & 1) * Smem::kStageBytes;
  }

  __device__ __forceinline__ void init() const {
    if (threadIdx.x == 0) {
      for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
      if constexpr (kRelease)
        for (int i = 3; i < 5; ++i) mbar_init(&bar[i], 2);  // one arrive per warpgroup
      fence_barrier_init();
    }
    __syncthreads();
  }
  // step n into stage s = n & 1
  template <class Load>
  __device__ __forceinline__ void load(uint32_t n, uint32_t s, const Load &issue) const {
    mbar_arrive_expect_tx(&bar[1 + s], Smem::kStageBytes);
    issue(n, stage(s), &bar[1 + s]);
  }
  // thread 0: the resident tiles (load_resident(base, bar)) and the first two steps
  template <class Resident, class Load>
  __device__ __forceinline__ void start(const Resident &load_resident, uint32_t total, const Load &load) const {
    if (threadIdx.x != 0) return;
    mbar_arrive_expect_tx(&bar[0], Smem::kResidentBytes);
    load_resident(base, &bar[0]);
    for (uint32_t n = 0; n < 2 && n < total; ++n) this->load(n, n, load);
  }
  __device__ __forceinline__ void wait_resident() const { mbar_wait(&bar[0], 0); }
  __device__ __forceinline__ void wait(uint32_t n) const { mbar_wait(&bar[1 + (n & 1)], (n >> 1) & 1); }
  // every thread is done with step n: its stage takes step n + 2
  template <class Load>
  __device__ __forceinline__ void release_and_refill(uint32_t n, uint32_t total, const Load &load) const {
    __syncthreads();
    if (threadIdx.x == 0 && n + 2 < total) this->load(n + 2, n & 1, load);
  }
  // kRelease: this warpgroup is done with step n (one thread: its wgmma_wait retired the warpgroup's wgmmas, and with
  // them their reads of the stage)
  __device__ __forceinline__ void release(uint32_t n) const {
    if (threadIdx.x % kWG == 0) mbar_arrive(&bar[3 + (n & 1)]);
  }
  // kRelease, thread 0: step n + 2 into the stage of step n once both warpgroups have released it
  template <class Load>
  __device__ __forceinline__ void refill(uint32_t n, uint32_t total, const Load &load) const {
    if (threadIdx.x == 0 && n + 2 < total) {
      mbar_wait(&bar[3 + (n & 1)], (n >> 1) & 1);
      this->load(n + 2, n & 1, load);
    }
  }
};

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

// Packed sequences: rows [first, ROWS) of a streamed DCH-chunk tile lie past the sequence's end, so TMA filled them with
// the next sequence's rows.  Zeroes them (each row is one 128-byte line of every chunk, whatever the swizzle): a masked
// product is 0 x x, which is NaN when x is not finite.  The caller fences and synchronises, as for the dO conversion.
template <uint32_t DCH, uint32_t ROWS, uint32_t kThreads>
__device__ __forceinline__ void zero_rows(uint8_t *tile, uint32_t first) {
  const uint32_t units = (ROWS - first) * 8;  // 16-byte units per chunk
  for (uint32_t i = threadIdx.x; i < DCH * units; i += kThreads) {
    const uint32_t c = i / units;
    reinterpret_cast<uint4 *>(tile + c * ROWS * 128 + first * 128)[i - c * units] = make_uint4(0u, 0u, 0u, 0u);
  }
}
// zero_rows of the rows [first, end)
template <uint32_t DCH, uint32_t ROWS, uint32_t kThreads>
__device__ __forceinline__ void zero_row_range(uint8_t *tile, uint32_t first, uint32_t end) {
  const uint32_t units = (end - first) * 8;
  for (uint32_t i = threadIdx.x; i < DCH * units; i += kThreads) {
    const uint32_t c = i / units;
    reinterpret_cast<uint4 *>(tile + c * ROWS * 128 + first * 128)[i - c * units] = make_uint4(0u, 0u, 0u, 0u);
  }
}

// FP32 accumulator rows -> global [rows][D] (row-major), columns < D, rows < limit
template <int NR>
__device__ __forceinline__ void store_acc(const float (&acc)[NR], float *out, uint32_t row0, uint32_t limit, uint32_t col0,
                                          uint32_t D, float inv0, float inv1) {
  const uint32_t t = threadIdx.x % kWG;
  const uint32_t r = row0 + frag_row(t);
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

// ================================================================================================ traversal ranges
// The key blocks of a forward / dQ CTA: [kb0, kb0 + result) of the split range [kb0, kb0 + per_split).  Causal: only
// those the rows [row_base, min(row_base + rows, R)) can see (key j <= row + delta).  Signed: a split range can lie
// wholly past the diagonal, and with R > C a tile can see no key at all.
template <uint32_t BN, bool kCausal>
__device__ __forceinline__ uint32_t key_blocks(uint32_t row_base, uint32_t rows, uint32_t R, uint32_t C, int delta,
                                               uint32_t kb0, uint32_t per_split) {
  if constexpr (!kCausal) {
    return min((C + BN - 1) / BN - kb0, per_split);
  } else {
    const int last_key = static_cast<int>(min(row_base + rows, R)) - 1 + delta;  // seen by the tile's last row
    const int end = last_key < 0 ? 0 : min(static_cast<int>((C + BN - 1) / BN), last_key / static_cast<int>(BN) + 1);
    return static_cast<uint32_t>(max(0, min(end, static_cast<int>(kb0 + per_split)) - static_cast<int>(kb0)));
  }
}

// Causal dK/dV: the first query block that sees key `key` (query >= key - delta), and how many of the blocks [qs, qb0 +
// per_split) exist (signed: a split range can end before qs)
template <uint32_t BM>
__device__ __forceinline__ uint32_t first_query_block(uint32_t key, int delta) {
  const int q = static_cast<int>(key) - delta;
  return q <= 0 ? 0u : static_cast<uint32_t>(q) / BM;
}
template <uint32_t BM>
__device__ __forceinline__ uint32_t visible_query_blocks(uint32_t R, uint32_t qb0, uint32_t qs, uint32_t per_split) {
  const int end = min(static_cast<int>((R + BM - 1) / BM), static_cast<int>(qb0 + per_split));
  return static_cast<uint32_t>(max(0, end - static_cast<int>(qs)));
}

// Sliding window: the blocks [first, end) of `block` rows of the axis of `length` rows that meet [lo, hi] (empty when
// end <= first)
template <uint32_t BLOCK>
__device__ __forceinline__ int2 band_blocks(int64_t lo, int64_t hi, uint32_t length) {
  const int first = lo <= 0 ? 0 : static_cast<int>(min(lo, static_cast<int64_t>(length)) / BLOCK);
  const int end = hi < 0 ? 0 : static_cast<int>(min(hi / BLOCK + 1, static_cast<int64_t>((length + BLOCK - 1) / BLOCK)));
  return make_int2(first, end);
}
// Forward / dQ: the key blocks the rows [row_base, min(row_base + rows, R)) see, keys [row_base + delta - left,
// last row + delta + right]
template <uint32_t BN>
__device__ __forceinline__ int2 band_key_blocks(uint32_t row_base, uint32_t rows, uint32_t R, uint32_t C, int delta,
                                                const Band &band) {
  const int64_t last = static_cast<int64_t>(min(row_base + rows, R)) - 1;
  return band_blocks<BN>(static_cast<int64_t>(row_base) + delta - band.left, last + delta + band.right, C);
}
// dK/dV: the query blocks that see the keys [key_base, min(key_base + keys, C)), queries [key_base - delta - right,
// last key - delta + left]
template <uint32_t BM>
__device__ __forceinline__ int2 band_query_blocks(uint32_t key_base, uint32_t keys, uint32_t R, uint32_t C, int delta,
                                                  const Band &band) {
  const int64_t last = static_cast<int64_t>(min(key_base + keys, C)) - 1;
  return band_blocks<BM>(static_cast<int64_t>(key_base) - delta - band.right, last - delta + band.left, R);
}
// The blocks of a CTA: the visible range [first, end) cut into split ranges of per_split blocks counted from `first`;
// *start receives the CTA's first block
__device__ __forceinline__ uint32_t band_split(int2 range, uint32_t split, uint32_t per_split, uint32_t *start) {
  *start = static_cast<uint32_t>(range.x) + split * per_split;
  return static_cast<uint32_t>(max(0, min(range.y, static_cast<int>(*start + per_split)) - static_cast<int>(*start)));
}

// ================================================================================================ masks
// Causal: a block whose last key is `last_key` has elements past the diagonal for some row from `first_query` on
__device__ __forceinline__ bool crosses_diagonal(int last_key, int first_query, int delta) {
  return last_key > first_query + delta;
}

// Causal: -inf for the elements past the diagonal (key > query + delta) of a 64 x N accumulator block, S (rows are
// queries, columns keys) or, kKeyRows, S^T (rows are keys, columns queries).  row: this thread's first row (the second
// is row + 8); col0: the block's first column.
template <bool kKeyRows, int NR>
__device__ __forceinline__ void mask_past_diagonal(float (&s)[NR], int row, int col0, int delta) {
  // masked: key > query + delta, with delta added to the query side (the columns of S^T, the row of S)
  const int c0 = col0 + 2 * static_cast<int>(threadIdx.x % 4) + (kKeyRows ? delta : 0);
  const int r0 = row + (kKeyRows ? 0 : delta);
#pragma unroll
  for (int i = 0; i < NR / 4; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = c0 + 8 * i + e;
      if (kKeyRows ? r0 > c : c > r0) s[4 * i + e] = -INFINITY;
      if (kKeyRows ? r0 + 8 > c : c > r0 + 8) s[4 * i + 2 + e] = -INFINITY;
    }
}

// Sliding window: -inf for the elements outside the band (query + lower <= key <= query + upper; lower = delta - left,
// upper = delta + right) of a 64 x N accumulator block, S (rows are queries, columns keys) or, kKeyRows, S^T (rows are
// keys, columns queries); row and col0 as for mask_past_diagonal.  Each row's band of columns is formed in 64 bits and
// clamped to the column range, so that neither a window side nor an index can overflow.
__device__ __forceinline__ int clamp_column(int64_t c) {
  return static_cast<int>(min(max(c, int64_t(-1)), static_cast<int64_t>(INT32_MAX)));
}
template <bool kKeyRows, int NR>
__device__ __forceinline__ void mask_outside_band(float (&s)[NR], int row, int col0, int64_t lower, int64_t upper) {
  int first[2], last[2];  // the columns [first, last] this thread's two rows keep
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t r = static_cast<int64_t>(row) + 8 * h;
    first[h] = clamp_column(kKeyRows ? r - upper : r + lower);
    last[h] = clamp_column(kKeyRows ? r - lower : r + upper);
  }
  const int c0 = col0 + 2 * static_cast<int>(threadIdx.x % 4);
#pragma unroll
  for (int i = 0; i < NR / 4; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = c0 + 8 * i + e;
      if (c < first[0] || c > last[0]) s[4 * i + e] = -INFINITY;
      if (c < first[1] || c > last[1]) s[4 * i + 2 + e] = -INFINITY;
    }
}
// mask_outside_band of S for a thread whose two rows are the query rows row0 and row1 (not row0 + 8: a tile that
// packs several query heads, forward_body's kSplit)
template <int NR>
__device__ __forceinline__ void mask_rows_outside_band(float (&s)[NR], int row0, int row1, int col0, int64_t lower,
                                                       int64_t upper) {
  const int first0 = clamp_column(row0 + lower), last0 = clamp_column(row0 + upper);
  const int first1 = clamp_column(row1 + lower), last1 = clamp_column(row1 + upper);
  const int c0 = col0 + 2 * static_cast<int>(threadIdx.x % 4);
#pragma unroll
  for (int i = 0; i < NR / 4; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = c0 + 8 * i + e;
      if (c < first0 || c > last0) s[4 * i + e] = -INFINITY;
      if (c < first1 || c > last1) s[4 * i + 2 + e] = -INFINITY;
    }
}
// Sliding window: whether a block of keys [key_first, key_last] x queries [query_first, query_last] crosses an edge of
// the band (64-bit, as mask_outside_band)
__device__ __forceinline__ bool crosses_band(int key_first, int key_last, int query_first, int query_last,
                                             int64_t lower, int64_t upper) {
  return key_last > query_first + upper || key_first < query_last + lower;
}

// Keys past C: -inf in both rows of a 64 x N accumulator block of S whose first key column is key0
template <int NR>
__device__ __forceinline__ void mask_past_edge(float (&s)[NR], uint32_t key0, uint32_t C) {
  const uint32_t c0 = key0 + 2 * (threadIdx.x % 4);
#pragma unroll
  for (uint32_t i = 0; i < NR / 4; ++i)
#pragma unroll
    for (uint32_t e = 0; e < 2; ++e)
      if (c0 + 8 * i + e >= C) s[4 * i + e] = s[4 * i + 2 + e] = -INFINITY;
}

// ================================================================================================ forward
// Split-KV (few query tiles for 132 SMs): the key axis of every tile is cut into `splits` equal ranges handled by
// separate CTAs (blockIdx.z), each leaving a normalised partial O and its log2-sum-exp in the library's workspace,
// laid out [split][head][row].  merge_splits, a second launch, merges the partials.
struct SplitArgs {
  uint32_t blocks_per_split, splits, batch;
  float *O_part, *L_part;  // [split][head][R][D], [split][head][R]
};

// O[row][4 quad ..] and L[row] from the partials of every split (row = head * R + r): one thread per (row, 4 columns).
// Causal: a split that saw no key of a row left L = -inf (weight 0); a row that no split saw gets O = 0, L = +inf.
template <bool kCausal>
__device__ __forceinline__ void merge_row(const SplitArgs &sp, float *O, void *L, int l_prec, uint64_t rows_total,
                                          uint32_t D, uint64_t row, uint32_t quad) {
  float lmax = -INFINITY;
  for (uint32_t s = 0; s < sp.splits; ++s) lmax = fmaxf(lmax, __ldcg(sp.L_part + s * rows_total + row));
  const float lref = kCausal && lmax == -INFINITY ? 0.f : lmax;
  float denom = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (uint32_t s = 0; s < sp.splits; ++s) {
    const float w = exp2f(__ldcg(sp.L_part + s * rows_total + row) - lref);
    const float4 v = __ldcg(reinterpret_cast<const float4 *>(sp.O_part + (s * rows_total + row) * D) + quad);
    denom += w;
    acc.x = fmaf(w, v.x, acc.x);
    acc.y = fmaf(w, v.y, acc.y);
    acc.z = fmaf(w, v.z, acc.z);
    acc.w = fmaf(w, v.w, acc.w);
  }
  const bool empty = kCausal && denom == 0.f;
  const float inv = empty ? 0.f : 1.0f / denom;
  *reinterpret_cast<float4 *>(O + row * D + 4 * quad) = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
  if (quad == 0) store_stat(L, row, l_prec, empty ? INFINITY : lmax + log2f(denom));
}
template <bool kCausal>
__global__ void __launch_bounds__(128) merge_splits(const SplitArgs sp, float *O, void *L, int l_prec, uint64_t rows_total,
                                                    uint32_t D) {
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t row = idx / (D / 4);
  if (row >= rows_total) return;
  merge_row<kCausal>(sp, O, L, l_prec, rows_total, D, row, static_cast<uint32_t>(idx % (D / 4)));
}

// merge_splits of a split packed or paged forward: grid (row chunks of the longest sequence, heads, sequences); the
// sequence's rows come from row_offsets, clamped into [0, R] as the forward clamps them, and only rows inside the
// sequence are written.  Always empty-aware: a sequence without keys, or a row whose band misses a chunk, leaves
// L = -inf partials without a causal mask.
__global__ void __launch_bounds__(128) merge_sequence_splits(const SplitArgs sp, float *O, void *L, int l_prec,
                                                             uint32_t R, uint32_t D, const int32_t *row_offsets) {
  uint32_t q0;
  const uint32_t rows = sequence_rows(row_offsets, blockIdx.z, R, &q0);
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x, r = idx / (D / 4);
  if (r >= rows) return;
  merge_row<true>(sp, O, L, l_prec, static_cast<uint64_t>(sp.batch) * R, D, static_cast<uint64_t>(blockIdx.y) * R + q0 + r,
                  static_cast<uint32_t>(idx % (D / 4)));
}

// kPar / kTrav: rows of the parallelization / traversal axis per CTA / per pipeline stage; kQueryBoxRows /
// kKeyBoxRows: rows of the TMA boxes of Q and dO / of K and V; Smem: the shared-memory layout (every *Cfg has them)
template <uint32_t DCH>
struct FwdCfg {
  static constexpr uint32_t kThreads = 2 * kWG, kTileM = 2 * kRows, BN = DCH == 4 ? 64 : 128;
  static constexpr uint32_t kPar = kTileM, kTrav = BN, kQueryBoxRows = kTileM, kKeyBoxRows = BN;
  static constexpr uint32_t kQBytes = DCH * kTileM * 128, kKVBytes = DCH * BN * 128;
  using Smem = SmemLayout<kQBytes, kKVBytes>;  // resident Q; stage: K, V
  // FP8 K/V: resident Q; a ring stage holds the FP8 K and V blocks as TMA lands them, [chunk][BN][64] bytes each,
  // unswizzled; after the two stages, one converted stage of 16-bit K and V tiles laid out as Smem's; the same bytes
  static constexpr uint32_t kFp8Bytes = DCH * BN * 64;
  struct Fp8Smem {
    static constexpr uint32_t kResidentBytes = kQBytes, kStageBytes = 2 * kFp8Bytes;
    static constexpr uint32_t kConvertedOffset = kQBytes + 2 * kStageBytes;
    static constexpr uint32_t kBarOffset = kConvertedOffset + 2 * kKVBytes;
    static constexpr uint32_t kSmemBytes = 1024 + kBarOffset + kBarBytes;
  };
  static_assert(Fp8Smem::kSmemBytes == Smem::kSmemBytes, "FP8 K/V keeps the 16-bit kernels' shared memory");
};

// Where the forward's keys come from: every problem's [C][D] rows (kFixed), a packed sequence's rows of them
// (kPacked), or a sequence's pages of the K / V pools (kPaged)
enum class KVLayout { kFixed, kPacked, kPaged };

// Paged K/V: the TMA boxes of key block `block` into the DCH-chunk K tile at dst and the V tile `kv_bytes` after it,
// `box` rows each (min(P, BN)).  P >= BN: one box per chunk and tensor, at the block's page.  P < BN: the page ids of
// every box are read first, so that their loads overlap, then each box is issued for K and V.  Boxes that start at or
// past the sequence's C never read the page table: they load pool row 0, and the caller zeroes every row past C before
// the MMAs.  ROW: bytes of one tile row of a chunk (128: 64 16-bit elements; 64: 64 FP8 bytes).
template <uint32_t DCH, uint32_t BN, uint32_t ROW = 128>
__device__ __forceinline__ void load_paged_kv(uint8_t *dst, uint32_t kv_bytes, const CUtensorMap *mapK,
                                              const CUtensorMap *mapV, uint64_t *bar, const PagedKV &pk,
                                              const int32_t *table, uint32_t block, uint32_t box, uint32_t C,
                                              uint32_t kv_head) {
  if (box == BN) {  // (a streamed block starts below C)
    const uint32_t row = paged_row(pk, table, block * BN);
#pragma unroll
    for (uint32_t c = 0; c < DCH; ++c) {
      tma_load_3d(dst + c * BN * ROW, mapK, bar, c * 64, kv_head, row);
      tma_load_3d(dst + kv_bytes + c * BN * ROW, mapV, bar, c * 64, kv_head, row);
    }
    return;
  }
  constexpr uint32_t kMaxBoxes = BN / 16;  // P >= 16
  uint32_t rows[kMaxBoxes];
#pragma unroll
  for (uint32_t i = 0; i < kMaxBoxes; ++i) {
    const uint32_t key = block * BN + i * box;
    rows[i] = i * box < BN && key < C ? paged_row(pk, table, key) : 0u;
  }
#pragma unroll
  for (uint32_t i = 0; i < kMaxBoxes; ++i) {
    if (i * box >= BN) break;
#pragma unroll
    for (uint32_t c = 0; c < DCH; ++c) {
      tma_load_3d(dst + c * BN * ROW + i * box * ROW, mapK, bar, c * 64, kv_head, rows[i]);
      tma_load_3d(dst + kv_bytes + c * BN * ROW + i * box * ROW, mapV, bar, c * 64, kv_head, rows[i]);
    }
  }
}

// Sliding window over a paged cache: the boxes of key block `block` that hold a key of [lo, hi] (the keys some row of
// the tile sees, within [0, C)), as [first, end) box indices
__device__ __forceinline__ uint2 band_boxes(uint32_t block, uint32_t BN, uint32_t box, int lo, int hi) {
  const int key0 = static_cast<int>(block * BN);
  const int first = max(lo - key0, 0) / static_cast<int>(box);
  const int end = min(hi - key0, static_cast<int>(BN) - 1) / static_cast<int>(box) + 1;
  return make_uint2(static_cast<uint32_t>(first), static_cast<uint32_t>(end));
}
// load_paged_kv of a windowed tile: only the boxes band_boxes names are issued, so the page-table entries and pages of
// the others are never read; the bytes they would have brought are completed on `bar` by hand, and the caller zeroes
// their rows
template <uint32_t DCH, uint32_t BN, uint32_t ROW = 128>
__device__ __forceinline__ void load_paged_kv_band(uint8_t *dst, uint32_t kv_bytes, const CUtensorMap *mapK,
                                                   const CUtensorMap *mapV, uint64_t *bar, const PagedKV &pk,
                                                   const int32_t *table, uint32_t block, uint32_t box, int lo, int hi,
                                                   uint32_t kv_head) {
  const uint2 kept = band_boxes(block, BN, box, lo, hi);
  constexpr uint32_t kMaxBoxes = BN / 16;  // P >= 16
  uint32_t rows[kMaxBoxes];
#pragma unroll
  for (uint32_t i = 0; i < kMaxBoxes; ++i)
    rows[i] = i >= kept.x && i < kept.y ? paged_row(pk, table, block * BN + i * box) : 0u;
  const uint32_t skipped = BN / box - (kept.y - kept.x);
  if (skipped) mbar_complete_tx(bar, skipped * box * ROW * DCH * 2);
#pragma unroll
  for (uint32_t i = 0; i < kMaxBoxes; ++i) {
    if (i < kept.x || i >= kept.y) continue;
#pragma unroll
    for (uint32_t c = 0; c < DCH; ++c) {
      tma_load_3d(dst + c * BN * ROW + i * box * ROW, mapK, bar, c * 64, kv_head, rows[i]);
      tma_load_3d(dst + kv_bytes + c * BN * ROW + i * box * ROW, mapV, bar, c * 64, kv_head, rows[i]);
    }
  }
}

// FP8 K/V: the landed block at src (FP8 K then V, [chunk][BN][64] bytes each) converted into the 16-bit K and V tiles
// at dst ([chunk][BN][64] elements, 128-byte swizzled, as TMA writes them for the 16-bit kernels).  Rows outside
// [first, end) -- past the sequence's keys, or in boxes that were not issued -- are written as zeros instead: a masked
// product is 0 x x, which is NaN when x is not finite.  The caller fences and synchronises.
template <uint32_t DCH, uint32_t BN, uint32_t kThreads, bool kBF16>
__device__ __forceinline__ void convert_fp8_kv(const uint8_t *src, uint8_t *dst, uint32_t first, uint32_t end) {
  // 16-byte units of the landed block: i = ((tensor * DCH + chunk) * BN + row) * 4 + quarter, at byte 16 i; its 16
  // elements go to 16-byte units 2 quarter and 2 quarter + 1 of line i / 4 of dst, each XORed with row % 8
  constexpr uint32_t kUnits = 2 * DCH * BN * 4;
  static_assert(kUnits % kThreads == 0, "every thread converts the same number of units");
#pragma unroll 4
  for (uint32_t i = threadIdx.x; i < kUnits; i += kThreads) {
    const uint32_t row = (i / 4) % BN, quarter = i % 4;
    uint4 lo = make_uint4(0u, 0u, 0u, 0u), hi = lo;
    if (row >= first && row < end) {
      const uint4 v = *reinterpret_cast<const uint4 *>(src + 16 * i);
      const uint2 a = e4m3x4_to_f16x4(v.x), b = e4m3x4_to_f16x4(v.y), c = e4m3x4_to_f16x4(v.z),
                  d = e4m3x4_to_f16x4(v.w);
      lo = make_uint4(a.x, a.y, b.x, b.y);
      hi = make_uint4(c.x, c.y, d.x, d.y);
      if constexpr (kBF16) {
        lo = make_uint4(f16x2_to_bf16x2(lo.x), f16x2_to_bf16x2(lo.y), f16x2_to_bf16x2(lo.z), f16x2_to_bf16x2(lo.w));
        hi = make_uint4(f16x2_to_bf16x2(hi.x), f16x2_to_bf16x2(hi.y), f16x2_to_bf16x2(hi.z), f16x2_to_bf16x2(hi.w));
      }
    }
    uint8_t *line = dst + (i / 4) * 128;
    *reinterpret_cast<uint4 *>(line + ((2 * quarter) ^ (row % 8)) * 16) = lo;
    *reinterpret_cast<uint4 *>(line + ((2 * quarter + 1) ^ (row % 8)) * 16) = hi;
  }
}

// The arguments of every forward kernel but its tensor maps.  Each kernel reads the fields its form uses:
//   O, L, l_prec   the outputs (O FP32 [batch][R][D], L [batch][R] in precision l_prec)
//   R, C, D        the rows of each problem's buffers (paged: C is unused) and the head dimension
//   delta          fixed-length problems: query row i sees key j iff j <= i + delta (C - R), the window's centre
//   group          query heads per K/V head
//   sp             the split of the key range and the workspace of its partials (the unsplit packed and paged kernels
//                  ignore it: they are never split)
//   hpt            split packed and paged kernels: query heads per tile
//   seq, pk        the packed sequences or the paged cache
//   band           the sliding window of the band_* kernels and their split and FP8 twins
//   fp8            the scales of FP8 pools
struct FwdArgs {
  float *O;
  void *L;
  uint32_t R, C, D;
  float scale_log2;
  int l_prec, delta;
  uint32_t group;
  SplitArgs sp;
  uint32_t hpt;
  Sequences seq;
  PagedKV pk;
  Band band;
  Fp8KV fp8;
};

// The body of the forward kernels.  kPacked / kPaged: the CTA works on sequence blockIdx.z, whose span replaces R, C
// and delta in the ranges and masks and offsets every query row, and zeroes the rows of its last key block past the
// sequence's keys.
// kBand: the sliding window `band` (with kCausal set).
// kSplit (packed / paged only): blockIdx.x is tile * sp.splits + split; the CTA takes chunk `split` of ceil(n / splits)
// blocks of the n key blocks its tile sees in its own sequence, and leaves a partial (an empty chunk: O = 0, L = -inf)
// at [split][head][packed row] of the workspace for merge_sequence_splits (one split: O and L themselves).  Its tile
// holds m = kTileM / hpt query rows of each of the hpt query heads blockIdx.y * hpt + [0, hpt) (hpt = 1, or the K/V
// group): tile row t is head blockIdx.y * hpt + t / m, query row tile * m + t % m; rows hpt * m .. kTileM - 1 are never
// stored.  Each row is masked with its own query row, so its arithmetic is that of the unpacked tile.
// kFp8 (kSplit paged only): the pools hold E4M3 bytes (mapK / mapV are 8-bit page-pool maps).  The ring lands each FP8
// block (Cfg::Fp8Smem); the threads convert it into the one 16-bit stage, zeroing the rows the 16-bit path zeroes, and
// the MMAs read that stage.  fp8.k_scale[kv_head] multiplies scale_log2, fp8.v_scale[kv_head] the epilogue's 1 / l.
template <uint32_t DCH, bool kBF16, bool kCausal, KVLayout kLayout, bool kBand = false, bool kSplit = false,
          bool kFp8 = false>
__device__ __forceinline__ void forward_body(const CUtensorMap &mapQ, const CUtensorMap &mapK, const CUtensorMap &mapV,
                                             const FwdArgs &a) {
  constexpr bool kVarlen = kLayout != KVLayout::kFixed;
  static_assert(!kSplit || kVarlen, "the fixed-length forward splits through blockIdx.z");
  static_assert(!kFp8 || (kSplit && kLayout == KVLayout::kPaged), "FP8 K/V is a split paged forward");
  float *__restrict__ O = a.O;
  void *__restrict__ L = a.L;
  const uint32_t R = a.R, C = a.C, D = a.D, group = a.group, hpt = a.hpt;
  const int l_prec = a.l_prec;
  const Sequences &seq = a.seq;
  const PagedKV &pk = a.pk;
  const Band &band = a.band;
  const Fp8KV &fp8 = a.fp8;
  const SplitArgs sp = kVarlen && !kSplit ? SplitArgs{0, 1, 0, nullptr, nullptr} : a.sp;
  float scale_log2 = a.scale_log2;
  int delta = a.delta;
  using Cfg = FwdCfg<DCH>;
  constexpr uint32_t NO = DCH * 64, BN = Cfg::BN;
  extern __shared__ uint8_t smem_raw[];
  using Smem = std::conditional_t<kFp8, typename Cfg::Fp8Smem, typename Cfg::Smem>;
  // the unmasked fixed-length forward has no CTA-wide barrier in its key loop (Ring's kRelease)
  constexpr bool kRelease = kLayout == KVLayout::kFixed && !kCausal;
  const Ring<Smem, kRelease> ring(smem_raw);  // resident Q; step j: K and V of key block kb0 + j
  const uint32_t tid = threadIdx.x, wg = tid / kWG, t = tid % kWG;
  const uint32_t tile = kSplit ? blockIdx.x / sp.splits : blockIdx.x;
  // (causal: unlike dQ, the forward gains nothing measurable from starting the tiles with the most key blocks first)
  const uint32_t tile_rows = kSplit ? Cfg::kTileM / hpt : Cfg::kTileM;  // query rows of each head in the tile (m)
  const uint32_t head = blockIdx.y, row_base = tile * tile_rows;
  // grouped K/V: the query heads of a group read one K/V head (kSplit: the tile's heads start at head * hpt)
  const uint32_t kv_head = (kSplit ? head * hpt : head) / group;
  float v_scale = 1.f;
  if constexpr (kFp8) {
    if (fp8.k_scale) scale_log2 *= __ldg(fp8.k_scale + kv_head);
    if (fp8.v_scale) v_scale = __ldg(fp8.v_scale + kv_head);
  }
  SequenceSpan span{0, R, 0, C};
  uint32_t kb0, per_split;
  if constexpr (kVarlen) {
    span = kLayout == KVLayout::kPaged ? paged_span(pk, blockIdx.z) : sequence_span(seq, blockIdx.z);
    if (row_base >= span.R) return;  // a tile past the sequence's end
    delta = static_cast<int>(span.C) - static_cast<int>(span.R);
    kb0 = 0;
    per_split = (span.C + BN - 1) / BN;
  } else {
    kb0 = blockIdx.z * sp.blocks_per_split;
    per_split = sp.blocks_per_split;
  }
  uint32_t blocks;
  if constexpr (kSplit) {
    // the visible blocks [first, end) of the tile in its sequence, cut by ceiling (a chunk may hold no block)
    const int2 range = kBand ? band_key_blocks<BN>(row_base, tile_rows, span.R, span.C, delta, band)
                             : make_int2(0, static_cast<int>(key_blocks<BN, kCausal>(row_base, tile_rows, span.R,
                                                                                     span.C, delta, 0, per_split)));
    const uint32_t n = static_cast<uint32_t>(max(range.y - range.x, 0));
    blocks = band_split(range, blockIdx.x % sp.splits, (n + sp.splits - 1) / sp.splits, &kb0);
  } else if constexpr (kBand) {
    blocks = band_split(band_key_blocks<BN>(row_base, Cfg::kTileM, span.R, span.C, delta, band),
                        kVarlen ? 0u : blockIdx.z, per_split, &kb0);
  } else {
    blocks = key_blocks<BN, kCausal>(row_base, Cfg::kTileM, span.R, span.C, delta, kb0, per_split);
  }
  // window: the keys [band_lo, band_hi] some row of the tile sees, clamped into [-1, C]
  const int64_t band_last = static_cast<int64_t>(min(row_base + tile_rows, span.R)) - 1;
  const int band_lo = kBand ? static_cast<int>(max(static_cast<int64_t>(row_base) + delta - band.left, int64_t(-1))) : 0;
  const int band_hi = kBand ? static_cast<int>(min(band_last + delta + band.right, static_cast<int64_t>(span.C))) : 0;

  // paged: this sequence's page_table row, and the rows of one TMA box
  const int32_t *table = kLayout == KVLayout::kPaged ? pk.page_table + static_cast<size_t>(blockIdx.z) * pk.page_stride
                                                     : nullptr;
  const uint32_t box = kLayout == KVLayout::kPaged ? min(1u << pk.page_shift, BN) : BN;
  auto load_kv = [&](uint32_t j, uint8_t *dst, uint64_t *bar) {
    if constexpr (kFp8 && kBand) {
      load_paged_kv_band<DCH, BN, 64>(dst, Cfg::kFp8Bytes, &mapK, &mapV, bar, pk, table, kb0 + j, box, band_lo,
                                      min(band_hi, static_cast<int>(span.C) - 1), kv_head);
    } else if constexpr (kFp8) {
      load_paged_kv<DCH, BN, 64>(dst, Cfg::kFp8Bytes, &mapK, &mapV, bar, pk, table, kb0 + j, box, span.C, kv_head);
    } else if constexpr (kLayout == KVLayout::kPaged && kBand) {
      load_paged_kv_band<DCH, BN>(dst, Cfg::kKVBytes, &mapK, &mapV, bar, pk, table, kb0 + j, box, band_lo,
                                  min(band_hi, static_cast<int>(span.C) - 1), kv_head);
    } else if constexpr (kLayout == KVLayout::kPaged) {
      load_paged_kv<DCH, BN>(dst, Cfg::kKVBytes, &mapK, &mapV, bar, pk, table, kb0 + j, box, span.C, kv_head);
    } else {
      load_tile<DCH, BN>(dst, &mapK, bar, span.k0 + (kb0 + j) * BN, kv_head);
      load_tile<DCH, BN>(dst + Cfg::kKVBytes, &mapV, bar, span.k0 + (kb0 + j) * BN, kv_head);
    }
  };
  if (tid == 0) {
    prefetch_tensormap(&mapQ);
    prefetch_tensormap(&mapK);
    prefetch_tensormap(&mapV);
  }
  ring.init();
  ring.start(
      [&](uint8_t *dst, uint64_t *bar) {
        // (kSplit: boxes of m rows x hpt heads; the rows past hpt * m are never loaded, their bytes completed by hand)
        load_tile<DCH, Cfg::kTileM>(dst, &mapQ, bar, span.q0 + row_base, kSplit ? head * hpt : head);
        if (kSplit && hpt * tile_rows < Cfg::kTileM) mbar_complete_tx(bar, (Cfg::kTileM - hpt * tile_rows) * 128 * DCH);
      },
      blocks, load_kv);

  const uint32_t sQ = smem_u32(ring.base);
  float o[NO / 2];
  zero(o);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  // kSplit: the tile rows of this thread (the second is 8 below the first) and their query rows
  const uint32_t trow0 = wg * kRows + frag_row(t);
  const int qrow0 = static_cast<int>(row_base + trow0 % tile_rows);
  const int qrow1 = static_cast<int>(row_base + (trow0 + 8) % tile_rows);
  ring.wait_resident();
  for (uint32_t j = 0; j < blocks; ++j) {
    ring.wait(j);
    if constexpr (kFp8) {
      // the rows [first, end) of the block that hold keys to use: below C, and (window) in the boxes that were issued
      uint32_t first = 0, end = min(BN, span.C - (kb0 + j) * BN);
      if constexpr (kBand) {
        const uint2 kept = band_boxes(kb0 + j, BN, box, band_lo, min(band_hi, static_cast<int>(span.C) - 1));
        first = kept.x * box;
        end = min(kept.y * box, end);
      }
      convert_fp8_kv<DCH, BN, Cfg::kThreads, kBF16>(ring.stage(j), ring.base + Cfg::Fp8Smem::kConvertedOffset, first, end);
      fence_proxy_async_smem();
      __syncthreads();
      // the landed block is spent: its stage takes step j + 2 while this block's MMAs run
      if (tid == 0 && j + 2 < blocks) ring.load(j + 2, j & 1, load_kv);
    } else if constexpr (kLayout == KVLayout::kPaged && kBand) {
      // the rows of the boxes that were not issued, and those past C
      const uint2 kept = band_boxes(kb0 + j, BN, box, band_lo, min(band_hi, static_cast<int>(span.C) - 1));
      const uint32_t first = kept.x * box, end = min(kept.y * box, span.C - (kb0 + j) * BN);
      if (first > 0 || end < BN) {
        zero_row_range<DCH, BN, Cfg::kThreads>(ring.stage(j), 0, first);
        zero_row_range<DCH, BN, Cfg::kThreads>(ring.stage(j), end, BN);
        zero_row_range<DCH, BN, Cfg::kThreads>(ring.stage(j) + Cfg::kKVBytes, 0, first);
        zero_row_range<DCH, BN, Cfg::kThreads>(ring.stage(j) + Cfg::kKVBytes, end, BN);
        fence_proxy_async_smem();
        __syncthreads();
      }
    } else if (kVarlen && ((kBand || kSplit ? kb0 : 0) + j + 1) * BN > span.C) {
      // the sequence's last key block: the next sequence's keys and values (packed), or whatever the page holds past C
      const uint32_t kb = (kBand || kSplit ? kb0 : 0) + j;
      zero_rows<DCH, BN, Cfg::kThreads>(ring.stage(j), span.C - kb * BN);
      zero_rows<DCH, BN, Cfg::kThreads>(ring.stage(j) + Cfg::kKVBytes, span.C - kb * BN);
      fence_proxy_async_smem();
      __syncthreads();
    }
    const uint32_t sK = smem_u32(kFp8 ? ring.base + Cfg::Fp8Smem::kConvertedOffset : ring.stage(j)), sV = sK + Cfg::kKVBytes;
    float sc[BN / 2];
    zero(sc);
    wgmma_fence();
    mma_ss<DCH, BN, kBF16, Cfg::kTileM>(sc, sQ, wg * kRows, sK);
    wgmma_commit();
    // kRelease: the stage of step j - 1 takes step j + 1 while this S product runs (thread 0 may wait there for the
    // other warpgroup to release it)
    if constexpr (kRelease)
      if (j > 0) ring.refill(j - 1, blocks, load_kv);
    wgmma_wait<0>();
    fence_regs(sc);

    // keys past C: -inf before the row max
    if ((kb0 + j + 1) * BN > span.C) mask_past_edge(sc, (kb0 + j) * BN, span.C);
    if constexpr (kSplit) {
      // each row against its own query row: causal is the band (-inf, delta]
      const int key0 = static_cast<int>((kb0 + j) * BN);
      const int64_t lower = kBand ? static_cast<int64_t>(delta) - band.left : -(int64_t(1) << 40);
      const int64_t upper = static_cast<int64_t>(delta) + (kBand ? band.right : 0);
      if ((kBand || kCausal) && crosses_band(key0, key0 + static_cast<int>(BN) - 1, static_cast<int>(row_base),
                                             static_cast<int>(row_base + tile_rows) - 1, lower, upper))
        mask_rows_outside_band(sc, qrow0, qrow1, key0, lower, upper);
    } else if constexpr (kBand) {
      const int key0 = static_cast<int>((kb0 + j) * BN), row = static_cast<int>(row_base + wg * kRows + frag_row(t));
      const int64_t lower = static_cast<int64_t>(delta) - band.left, upper = static_cast<int64_t>(delta) + band.right;
      if (crosses_band(key0, key0 + static_cast<int>(BN) - 1, static_cast<int>(row_base),
                       static_cast<int>(row_base + Cfg::kTileM) - 1, lower, upper))
        mask_outside_band<false>(sc, row, key0, lower, upper);
    } else if constexpr (kCausal) {
      const int key0 = static_cast<int>((kb0 + j) * BN);
      if (crosses_diagonal(key0 + static_cast<int>(BN) - 1, static_cast<int>(row_base), delta))
        mask_past_diagonal<false>(sc, static_cast<int>(row_base + wg * kRows + frag_row(t)), key0, delta);
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
    // causal: a row that has seen no key yet keeps m = -inf; 0 stands in for it as the reference value (else -inf - -inf)
    const float ref0 = kCausal && mn0 == -INFINITY ? 0.f : mn0, ref1 = kCausal && mn1 == -INFINITY ? 0.f : mn1;
    const float a0 = ex2_approx(m0 - ref0), a1 = ex2_approx(m1 - ref1);  // 0 on the first block (m = -inf)
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
      sc[4 * i] = ex2_approx(fmaf(sc[4 * i], scale_log2, -ref0));
      sc[4 * i + 1] = ex2_approx(fmaf(sc[4 * i + 1], scale_log2, -ref0));
      sc[4 * i + 2] = ex2_approx(fmaf(sc[4 * i + 2], scale_log2, -ref1));
      sc[4 * i + 3] = ex2_approx(fmaf(sc[4 * i + 3], scale_log2, -ref1));
      l0 += sc[4 * i] + sc[4 * i + 1];
      l1 += sc[4 * i + 2] + sc[4 * i + 3];
    }
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < BN / 16; ++kk) {
      uint32_t a[4];
      a_frag<kBF16>(sc, kk, a);
      Wgmma<NO, kBF16>::rs(o, a, desc_mnmajor<BN>(sV, kk, 0), 1);
      // D <= 64: retiring each K step before packing the next A fragment keeps the kernel within 128 registers, so
      // two CTAs share an SM (their shared memory fits twice); with every fragment in flight it takes 145 and one CTA
      // per SM, about 12 % slower
      if constexpr (DCH == 1) {
        wgmma_commit();
        wgmma_wait<0>();
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    if constexpr (kFp8)
      __syncthreads();  // every warpgroup is done with the converted stage: the next block may overwrite it
    else if constexpr (kRelease)
      ring.release(j);
    else
      ring.release_and_refill(j, blocks, load_kv);
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  if constexpr (kSplit) {
    // each of this thread's two rows at its own (head, query row); one split: O and L, else the partial of this range
    const uint32_t split = blockIdx.x % sp.splits;
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
      const uint32_t trow = trow0 + 8 * h, r = row_base + trow % tile_rows, qh = head * hpt + trow / tile_rows;
      if (trow >= hpt * tile_rows || r >= span.R) continue;
      const float l = h ? l1 : l0, mrow = h ? m1 : m0;
      // (FP8: times the V scale, which scales O and not L; a power of two keeps the product exact)
      const float inv = l == 0.f ? 0.f : (kFp8 ? (1.0f / l) * v_scale : 1.0f / l);
      const size_t row = (sp.splits == 1 ? static_cast<size_t>(qh) : static_cast<size_t>(split) * sp.batch + qh) * R +
                         span.q0 + r;
      float *out = (sp.splits == 1 ? O : sp.O_part) + row * D;
#pragma unroll
      for (int i = 0; i < NO / 8; ++i) {
        const uint32_t col = 8 * i + 2 * (t % 4);
        if (col < D)
          *reinterpret_cast<float2 *>(out + col) = make_float2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
      }
      if (t % 4 == 0)
        store_stat(sp.splits == 1 ? L : sp.L_part, row, sp.splits == 1 ? l_prec : FP32,
                   l == 0.f ? (sp.splits == 1 ? INFINITY : -INFINITY) : mrow + log2f(l));
    }
    return;
  }
  const uint32_t row0 = row_base + wg * kRows;
  // unsplit: O and L straight to the caller; split: the normalised partial of this key range
  const size_t slice = static_cast<size_t>(blockIdx.z) * sp.batch + head;
  float *Oout = sp.splits == 1 ? O + (static_cast<size_t>(head) * R + span.q0) * D : sp.O_part + slice * R * D;
  // causal, or a sequence without keys: a row that saw no key (l = 0) gets O = 0 and L = +inf, or L = -inf (weight 0 in
  // the merge) as a split partial
  const bool empty0 = (kCausal || kVarlen) && l0 == 0.f, empty1 = (kCausal || kVarlen) && l1 == 0.f;
  store_acc(o, Oout, row0, span.R, 0, D, empty0 ? 0.f : 1.0f / l0, empty1 ? 0.f : 1.0f / l1);
  if (t % 4 == 0) {
    const uint32_t r = row0 + frag_row(t);
    void *Lout = sp.splits == 1 ? L : sp.L_part;
    const int prec = sp.splits == 1 ? l_prec : FP32;
    const size_t hb = (sp.splits == 1 ? static_cast<size_t>(head) : slice) * R + span.q0;
    const float none = sp.splits == 1 ? INFINITY : -INFINITY;
    if (r < span.R) store_stat(Lout, hb + r, prec, empty0 ? none : m0 + log2f(l0));
    if (r + 8 < span.R) store_stat(Lout, hb + r + 8, prec, empty1 ? none : m1 + log2f(l1));
  }
}

// Fixed-length problems: grid (tiles, heads, splits); each split is one range of blocks_per_split key blocks, and
// with more than one, merge_splits merges the partials
template <uint32_t DCH, bool kBF16, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    attention_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                            const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, kCausal, KVLayout::kFixed>(mapQ, mapK, mapV, a);
}

// Packed sequences: grid (tiles of the longest sequence, heads, sequences)
template <uint32_t DCH, bool kBF16, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    packed_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                         const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, kCausal, KVLayout::kPacked>(mapQ, mapK, mapV, a);
}

// Paged K/V: grid (tiles of the longest query sequence, heads, sequences); mapK / mapV are page-pool maps
template <uint32_t DCH, bool kBF16, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    paged_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                        const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, kCausal, KVLayout::kPaged>(mapQ, mapK, mapV, a);
}

// Sliding window: the three forward kernels above with a band, causal or not (a causal window is a band with right = 0)
template <uint32_t DCH, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    band_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                       const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, true, KVLayout::kFixed, true>(mapQ, mapK, mapV, a);
}
template <uint32_t DCH, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    band_forward_packed_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                              const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, true, KVLayout::kPacked, true>(mapQ, mapK, mapV, a);
}
template <uint32_t DCH, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    band_forward_paged_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                             const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, true, KVLayout::kPaged, true>(mapQ, mapK, mapV, a);
}

// Split-KV packed and paged forwards (kSplit): grid (tiles of the longest query sequence x sp.splits, heads / hpt,
// sequences), hpt query heads per tile; with more than one split the partials are merged by merge_sequence_splits.
// Windowed twins with a band.
template <uint32_t DCH, bool kBF16, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    split_forward_packed_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                               const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, kCausal, KVLayout::kPacked, false, true>(mapQ, mapK, mapV, a);
}
// (D <= 64, not causal: held to two CTAs per SM, which its 127 registers allowed when its arguments were separate
// kernel parameters; read from one struct, ptxas would take 131 and one CTA.  It fits 128 without spilling.)
template <uint32_t DCH, bool kBF16, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, DCH == 1 && !kCausal ? 2 : 1)
    split_forward_paged_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                              const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, kCausal, KVLayout::kPaged, false, true>(mapQ, mapK, mapV, a);
}
template <uint32_t DCH, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    split_forward_packed_band_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                    const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, true, KVLayout::kPacked, true, true>(mapQ, mapK, mapV, a);
}
template <uint32_t DCH, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    split_forward_paged_band_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                   const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, true, KVLayout::kPaged, true, true>(mapQ, mapK, mapV, a);
}

// FP8 K/V: the two split paged forwards above over E4M3 pools with per-K/V-head scales (mapK / mapV: 8-bit page-pool
// maps).  An unsplit call runs them with one split and one head per tile.
template <uint32_t DCH, bool kBF16, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    fp8_kv_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                         const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, kCausal, KVLayout::kPaged, false, true, true>(mapQ, mapK, mapV, a);
}
template <uint32_t DCH, bool kBF16>
__global__ void __launch_bounds__(2 * kWG, 1)
    fp8_kv_window_forward_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                                const __grid_constant__ CUtensorMap mapV, const __grid_constant__ FwdArgs a) {
  forward_body<DCH, kBF16, true, KVLayout::kPaged, true, true, true>(mapQ, mapK, mapV, a);
}

// ================================================================================================ backward dQ
template <uint32_t DCH>
struct QCfg {
  static constexpr uint32_t kWarpgroups = DCH == 4 ? 1 : 2;
  static constexpr uint32_t kThreads = kWarpgroups * kWG, kTileM = kWarpgroups * kRows, BN = 64;
  static constexpr uint32_t kPar = kTileM, kTrav = BN, kQueryBoxRows = kTileM, kKeyBoxRows = BN;
  static constexpr uint32_t kQBytes = DCH * kTileM * 128, kKVBytes = DCH * BN * 128;
  using Smem = SmemLayout<2 * kQBytes, kKVBytes>;  // resident Q, dO; stage: K, V
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
  int delta;  // causal kernels: query row i sees key j iff j <= i + delta
  uint32_t group;  // query heads per K/V head: query head h reads K/V head h / group
};

// The body of the dQ kernels; kVarlen and kBand as in forward_body
template <uint32_t DCH, bool kBF16, bool kConvertDO, bool kCausal, bool kVarlen, bool kBand = false>
__device__ __forceinline__ void backward_query_body(const CUtensorMap &mapQ, const CUtensorMap &mapdO,
                                                    const CUtensorMap &mapK, const CUtensorMap &mapV, const BwdArgs &a,
                                                    const Sequences &seq, const Band &band) {
  using Cfg = QCfg<DCH>;
  constexpr uint32_t NO = DCH * 64, BN = Cfg::BN;
  extern __shared__ uint8_t smem_raw[];
  const Ring<typename Cfg::Smem> ring(smem_raw);  // resident Q, dO; step j: K and V of key block kb0 + j
  const uint32_t tid = threadIdx.x, wg = tid / kWG, t = tid % kWG;
  // causal: tiles in reverse order, so that the ones with the most key blocks start first and the wave tail is short
  const uint32_t tile = kCausal ? gridDim.x - 1 - blockIdx.x : blockIdx.x;
  const uint32_t head = blockIdx.y, row_base = tile * Cfg::kTileM, kv_head = head / a.group;
  SequenceSpan span{0, a.R, 0, a.C};
  int delta = a.delta;
  uint32_t kb0, per_split;
  if constexpr (kVarlen) {
    span = sequence_span(seq, blockIdx.z);
    if (row_base >= span.R) return;
    delta = static_cast<int>(span.C) - static_cast<int>(span.R);
    kb0 = 0;
    per_split = (span.C + BN - 1) / BN;
  } else {
    kb0 = blockIdx.z * a.blocks_per_split;
    per_split = a.blocks_per_split;
  }
  uint32_t blocks;
  if constexpr (kBand) {
    blocks = band_split(band_key_blocks<BN>(row_base, Cfg::kTileM, span.R, span.C, delta, band),
                        kVarlen ? 0u : blockIdx.z, per_split, &kb0);
  } else {
    blocks = key_blocks<BN, kCausal>(row_base, Cfg::kTileM, span.R, span.C, delta, kb0, per_split);
  }

  auto load_kv = [&](uint32_t j, uint8_t *dst, uint64_t *bar) {
    load_tile<DCH, BN>(dst, &mapK, bar, span.k0 + (kb0 + j) * BN, kv_head);
    load_tile<DCH, BN>(dst + Cfg::kKVBytes, &mapV, bar, span.k0 + (kb0 + j) * BN, kv_head);
  };
  ring.init();
  ring.start(
      [&](uint8_t *dst, uint64_t *bar) {
        load_tile<DCH, Cfg::kTileM>(dst, &mapQ, bar, span.q0 + row_base, head);
        load_tile<DCH, Cfg::kTileM>(dst + Cfg::kQBytes, &mapdO, bar, span.q0 + row_base, head);
      },
      blocks, load_kv);

  // D = rowsum(dO * O) / sqrt(D) for this thread's two rows (the four threads of a row split the columns), while the
  // tiles are in flight; stored for the dK/dV kernel, kept in FP32 here
  const uint32_t row0 = row_base + wg * kRows;
  const uint32_t r = row0 + frag_row(t);
  const size_t hb = static_cast<size_t>(head) * a.R + span.q0;
  float Dr[2], Lr[2];
#pragma unroll
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t rc = min(r + 8 * h, span.R - 1);
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
    if (t % 4 == 0 && r + 8 * h < span.R && (kVarlen || blockIdx.z == 0))
      store_stat(a.Dterm, hb + r + 8 * h, a.d_prec, Dr[h]);
  }

  const uint32_t sQ = smem_u32(ring.base), sdO = sQ + Cfg::kQBytes;
  ring.wait_resident();
  if constexpr (kConvertDO) {
    // BF16 dO beside FP16 Q/K/V: wgmma takes one element type for A and B, so the resident dO tile is rewritten as
    // FP16 in place (exact for 2^-14 <= |x| < 65504)
    uint4 *tile = reinterpret_cast<uint4 *>(ring.base + Cfg::kQBytes);
    for (uint32_t i = tid; i < Cfg::kQBytes / 16; i += Cfg::kThreads) tile[i] = bwd::bf16x8_to_f16x8(tile[i]);
    fence_proxy_async_smem();
    __syncthreads();
  }
  float dq[NO / 2];
  zero(dq);
  for (uint32_t j = 0; j < blocks; ++j) {
    ring.wait(j);
    if (kVarlen && ((kBand ? kb0 : 0) + j + 1) * BN > span.C) {  // the sequence's last key block: the next sequence's
      const uint32_t kb = (kBand ? kb0 : 0) + j;                  // keys and values
      zero_rows<DCH, BN, Cfg::kThreads>(ring.stage(j), span.C - kb * BN);
      zero_rows<DCH, BN, Cfg::kThreads>(ring.stage(j) + Cfg::kKVBytes, span.C - kb * BN);
      fence_proxy_async_smem();
      __syncthreads();
    }
    const uint32_t sK = smem_u32(ring.stage(j)), sV = sK + Cfg::kKVBytes;
    float sc[BN / 2], dp[BN / 2];
    zero(sc);
    zero(dp);
    wgmma_fence();
    mma_ss<DCH, BN, kBF16, Cfg::kTileM>(sc, sQ, wg * kRows, sK);
    mma_ss<DCH, BN, kBF16, Cfg::kTileM>(dp, sdO, wg * kRows, sV);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sc);
    fence_regs(dp);
    if constexpr (kBand) {  // S -> -inf outside the band, so P = 0 there
      const int key0 = static_cast<int>((kb0 + j) * BN);
      const int64_t lower = static_cast<int64_t>(delta) - band.left, upper = static_cast<int64_t>(delta) + band.right;
      if (crosses_band(key0, key0 + static_cast<int>(BN) - 1, static_cast<int>(row_base),
                       static_cast<int>(row_base + Cfg::kTileM) - 1, lower, upper))
        mask_outside_band<false>(sc, static_cast<int>(r), key0, lower, upper);
    } else if constexpr (kCausal) {  // S -> -inf past the diagonal, so P = 0 there
      const int key0 = static_cast<int>((kb0 + j) * BN);
      if (crosses_diagonal(key0 + static_cast<int>(BN) - 1, static_cast<int>(row_base), delta))
        mask_past_diagonal<false>(sc, static_cast<int>(r), key0, delta);
    }
    const uint32_t c0 = (kb0 + j) * BN + 2 * (t % 4);
#pragma unroll
    for (uint32_t i = 0; i < BN / 8; ++i)
#pragma unroll
      for (uint32_t e = 0; e < 4; ++e) {
        const uint32_t h = e >> 1, k = 4 * i + e;
        const float p = c0 + 8 * i + (e & 1) < span.C ? ex2_approx(fmaf(sc[k], a.scale_log2, -Lr[h])) : 0.f;
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
    ring.release_and_refill(j, blocks, load_kv);
  }
  store_acc(dq, a.dQ + (kVarlen ? 0 : blockIdx.z * a.split_stride) + hb * a.D, row0, span.R, 0, a.D, 1.f, 1.f);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO, bool kCausal>
__global__ void __launch_bounds__(QCfg<DCH>::kThreads, 1)
    attention_backward_query_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                   const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                   const BwdArgs a, const Sequences seq, const Band band) {
  backward_query_body<DCH, kBF16, kConvertDO, kCausal, false>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO, bool kCausal>
__global__ void __launch_bounds__(QCfg<DCH>::kThreads, 1)
    packed_backward_query_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                const BwdArgs a, const Sequences seq, const Band band) {
  backward_query_body<DCH, kBF16, kConvertDO, kCausal, true>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO>
__global__ void __launch_bounds__(QCfg<DCH>::kThreads, 1)
    band_backward_query_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                              const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                              const BwdArgs a, const Sequences seq, const Band band) {
  backward_query_body<DCH, kBF16, kConvertDO, true, false, true>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO>
__global__ void __launch_bounds__(QCfg<DCH>::kThreads, 1)
    band_backward_query_packed_wgmma(const __grid_constant__ CUtensorMap mapQ,
                                     const __grid_constant__ CUtensorMap mapdO,
                                     const __grid_constant__ CUtensorMap mapK,
                                     const __grid_constant__ CUtensorMap mapV, const BwdArgs a, const Sequences seq,
                                     const Band band) {
  backward_query_body<DCH, kBF16, kConvertDO, true, true, true>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

// ================================================================================================ backward dK/dV
template <uint32_t DCH>
struct KVCfg {
  static constexpr bool kSplitD = DCH == 4;  // both warpgroups on the same 64 keys, half of the D columns each
  static constexpr uint32_t kThreads = 2 * kWG, kTileN = kSplitD ? kRows : 2 * kRows, BM = 64;
  static constexpr uint32_t kPar = kTileN, kTrav = BM, kQueryBoxRows = BM, kKeyBoxRows = kTileN;
  static constexpr uint32_t kAcc = kSplitD ? 128 : DCH * 64;  // accumulator columns per warpgroup
  static constexpr uint32_t kKBytes = DCH * kTileN * 128, kQBytes = DCH * BM * 128;
  using Smem = SmemLayout<2 * kKBytes, kQBytes>;  // resident K, V; stage: Q, dO
};

// The body of the dK/dV kernels; kVarlen and kBand as in forward_body (a tile of keys whose sequence has no query, or
// that no query sees, stores zeros)
template <uint32_t DCH, bool kBF16, bool kConvertDO, bool kCausal, bool kVarlen, bool kBand = false>
__device__ __forceinline__ void backward_key_value_body(const CUtensorMap &mapQ, const CUtensorMap &mapdO,
                                                        const CUtensorMap &mapK, const CUtensorMap &mapV,
                                                        const BwdArgs &a, const Sequences &seq, const Band &band) {
  using Cfg = KVCfg<DCH>;
  constexpr uint32_t BM = Cfg::BM, NA = Cfg::kAcc;
  extern __shared__ uint8_t smem_raw[];
  const Ring<typename Cfg::Smem> ring(smem_raw);  // resident K, V; step n: Q and dO of one query block
  const uint32_t tid = threadIdx.x, wg = tid / kWG, t = tid % kWG;
  // grouped K/V: blockIdx.y is a K/V head, and the CTA walks the query blocks of every query head of its group
  const uint32_t kv_head = blockIdx.y, key_base = blockIdx.x * Cfg::kTileN;
  SequenceSpan span{0, a.R, 0, a.C};
  int delta = a.delta;
  uint32_t qb0, per_split;
  if constexpr (kVarlen) {
    span = sequence_span(seq, blockIdx.z);
    if (key_base >= span.C) return;
    delta = static_cast<int>(span.C) - static_cast<int>(span.R);
    qb0 = 0;
    per_split = (span.R + BM - 1) / BM;
  } else {
    qb0 = blockIdx.z * a.blocks_per_split;
    per_split = a.blocks_per_split;
  }
  uint32_t qs, blocks;
  if constexpr (kBand) {
    blocks = band_split(band_query_blocks<BM>(key_base, Cfg::kTileN, span.R, span.C, delta, band),
                        kVarlen ? 0u : blockIdx.z, per_split, &qs);
  } else {
    // causal: this CTA's query blocks start at the first one that sees the tile's first key (query >= key_base - delta)
    qs = kCausal ? max(qb0, first_query_block<BM>(key_base, delta)) : qb0;
    blocks = kCausal ? visible_query_blocks<BM>(span.R, qb0, qs, per_split) : min((span.R + BM - 1) / BM - qb0, per_split);
  }
  // the same query blocks [qs, qs + blocks) of each of the group's query heads, as one flattened sequence n = g blocks
  // + i that drives the Q / dO ring: prefetch and barrier parity carry across head boundaries
  const uint32_t total = a.group * blocks;

  auto load_qd = [&](uint32_t n, uint8_t *dst, uint64_t *bar) {
    const uint32_t g = n / blocks, i = n - g * blocks;
    load_tile<DCH, BM>(dst, &mapQ, bar, span.q0 + (qs + i) * BM, kv_head * a.group + g);
    load_tile<DCH, BM>(dst + Cfg::kQBytes, &mapdO, bar, span.q0 + (qs + i) * BM, kv_head * a.group + g);
  };
  ring.init();
  ring.start(
      [&](uint8_t *dst, uint64_t *bar) {
        load_tile<DCH, Cfg::kTileN>(dst, &mapK, bar, span.k0 + key_base, kv_head);
        load_tile<DCH, Cfg::kTileN>(dst + Cfg::kKBytes, &mapV, bar, span.k0 + key_base, kv_head);
      },
      total, load_qd);
  const uint32_t sK = smem_u32(ring.base), sV = sK + Cfg::kKBytes;
  const uint32_t krow = Cfg::kSplitD ? 0 : wg * kRows;      // this warpgroup's key rows inside the tile
  const uint32_t nchunk = Cfg::kSplitD ? wg * (NA / 64) : 0;  // ... and its first accumulator column chunk
  size_t hb = static_cast<size_t>(kv_head) * a.group * a.R + span.q0;  // L / D rows of the current query head
  float dv[NA / 2], dk[NA / 2];
  zero(dv);
  zero(dk);
  ring.wait_resident();
  for (uint32_t n = 0, i = 0; n < total; ++n) {
    // per-query statistics of this thread's 16 columns, loaded while the tiles land
    float Lq[BM / 4], Dq[BM / 4];
    const uint32_t q0 = (qs + i) * BM + 2 * (t % 4);
#pragma unroll
    for (uint32_t j = 0; j < BM / 8; ++j)
#pragma unroll
      for (uint32_t e = 0; e < 2; ++e) {
        const uint32_t q = min(q0 + 8 * j + e, span.R - 1);
        Lq[2 * j + e] = load_stat(a.L, hb + q, a.l_prec);
        Dq[2 * j + e] = load_stat(a.Dterm, hb + q, a.d_prec);
      }
    ring.wait(n);
    if constexpr (kConvertDO) {
      // BF16 dO beside FP16 Q/K/V on a small grid: the streamed dO tile is rewritten as FP16 in place (a grid of more
      // than one wave converts dO once, in a pass of its own, instead)
      uint4 *tile = reinterpret_cast<uint4 *>(ring.stage(n) + Cfg::kQBytes);
      for (uint32_t k = tid; k < Cfg::kQBytes / 16; k += Cfg::kThreads) tile[k] = bwd::bf16x8_to_f16x8(tile[k]);
      fence_proxy_async_smem();
      __syncthreads();
    }
    if (kVarlen && (qs + i + 1) * BM > span.R) {  // the sequence's last query block: the next sequence's Q and dO
      zero_rows<DCH, BM, Cfg::kThreads>(ring.stage(n), span.R - (qs + i) * BM);
      zero_rows<DCH, BM, Cfg::kThreads>(ring.stage(n) + Cfg::kQBytes, span.R - (qs + i) * BM);
      fence_proxy_async_smem();
      __syncthreads();
    }
    const uint32_t sQ = smem_u32(ring.stage(n)), sdO = sQ + Cfg::kQBytes;
    float st[BM / 2], dpt[BM / 2];
    zero(st);
    zero(dpt);
    wgmma_fence();
    mma_ss<DCH, BM, kBF16, Cfg::kTileN>(st, sK, krow, sQ);
    mma_ss<DCH, BM, kBF16, Cfg::kTileN>(dpt, sV, krow, sdO);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(st);
    fence_regs(dpt);
    if constexpr (kBand) {  // S^T -> -inf outside the band, so P^T = 0 there
      const int qlo = static_cast<int>((qs + i) * BM), key = static_cast<int>(key_base + krow + frag_row(t));
      const int64_t lower = static_cast<int64_t>(delta) - band.left, upper = static_cast<int64_t>(delta) + band.right;
      if (crosses_band(static_cast<int>(key_base), static_cast<int>(key_base + Cfg::kTileN) - 1, qlo,
                       qlo + static_cast<int>(BM) - 1, lower, upper))
        mask_outside_band<true>(st, key, qlo, lower, upper);
    } else if constexpr (kCausal) {  // S^T -> -inf where key > query + delta, so P^T = 0 there
      const int qlo = static_cast<int>((qs + i) * BM);
      if (crosses_diagonal(static_cast<int>(key_base + Cfg::kTileN) - 1, qlo, delta))
        mask_past_diagonal<true>(st, static_cast<int>(key_base + krow + frag_row(t)), qlo, delta);
    }
#pragma unroll
    for (uint32_t j = 0; j < BM / 8; ++j)
#pragma unroll
      for (uint32_t e = 0; e < 4; ++e) {
        const uint32_t k = 4 * j + e, c = 2 * j + (e & 1);
        const float p = q0 + 8 * j + (e & 1) < span.R ? ex2_approx(fmaf(st[k], a.scale_log2, -Lq[c])) : 0.f;
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
    ring.release_and_refill(n, total, load_qd);
    if (++i == blocks) {  // the next query head of the group; dK and dV keep accumulating
      i = 0;
      hb += a.R;
    }
  }
  const size_t kb = (static_cast<size_t>(kv_head) * a.C + span.k0) * a.D;
  const uint32_t row0 = key_base + krow, col0 = nchunk * 64;
  const size_t split = kVarlen ? 0 : blockIdx.z * a.split_stride;
  store_acc(dv, a.dV + split + kb, row0, span.C, col0, a.D, 1.f, 1.f);
  store_acc(dk, a.dK + split + kb, row0, span.C, col0, a.D, 1.f, 1.f);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    attention_backward_key_value_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                       const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                       const BwdArgs a, const Sequences seq, const Band band) {
  backward_key_value_body<DCH, kBF16, kConvertDO, kCausal, false>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO, bool kCausal>
__global__ void __launch_bounds__(2 * kWG, 1)
    packed_backward_key_value_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                    const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                    const BwdArgs a, const Sequences seq, const Band band) {
  backward_key_value_body<DCH, kBF16, kConvertDO, kCausal, true>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO>
__global__ void __launch_bounds__(2 * kWG, 1)
    band_backward_key_value_wgmma(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapdO,
                                  const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV,
                                  const BwdArgs a, const Sequences seq, const Band band) {
  backward_key_value_body<DCH, kBF16, kConvertDO, true, false, true>(mapQ, mapdO, mapK, mapV, a, seq, band);
}

template <uint32_t DCH, bool kBF16, bool kConvertDO>
__global__ void __launch_bounds__(2 * kWG, 1)
    band_backward_key_value_packed_wgmma(const __grid_constant__ CUtensorMap mapQ,
                                         const __grid_constant__ CUtensorMap mapdO,
                                         const __grid_constant__ CUtensorMap mapK,
                                         const __grid_constant__ CUtensorMap mapV, const BwdArgs a, const Sequences seq,
                                         const Band band) {
  backward_key_value_body<DCH, kBF16, kConvertDO, true, true, true>(mapQ, mapdO, mapK, mapV, a, seq, band);
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

// choose_splits of a split packed or paged forward, whose kernels cut each tile's visible key blocks by ceiling on the
// device: the bound need not divide evenly, and every range but the last has at least min_blocks of `total_blocks`
static uint32_t choose_key_splits(uint64_t items, uint32_t total_blocks, uint32_t sm_count, uint32_t min_blocks,
                                  uint32_t max_splits) {
  if (items * 2 > sm_count || min_blocks == 0) return 1;
  if (max_splits > 16) max_splits = 16;
  const uint32_t target = sm_count / static_cast<uint32_t>(items);
  uint32_t best = 1;
  for (uint32_t s = 2; s <= target && s <= max_splits; ++s)
    if (total_blocks / s >= min_blocks) best = s;
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

// Calls f(std::integral_constant<uint32_t, DCH>()) for the column-chunk count of the kernels that serve head dimension D
template <class F>
static auto with_chunks(uint32_t D, F f) {
  switch (chunks(D)) {
    case 1: return f(std::integral_constant<uint32_t, 1>());
    case 2: return f(std::integral_constant<uint32_t, 2>());
    default: return f(std::integral_constant<uint32_t, 4>());
  }
}

// ================================================================================================ launchers
template <typename Kernel>
static cudaError_t prepare(Kernel kernel, uint32_t smem) {
  return ensure_max_dynamic_smem(reinterpret_cast<const void *>(kernel), smem, current_device());
}

// The tensor maps of a backward kernel: Q and dO in boxes of query_rows rows, K and V in boxes of key_rows.  Grouped
// K/V: K and V hold batch / group heads.
struct TensorMaps {
  CUtensorMap Q, dO, K, V;
};
static cudaError_t make_maps(const AttentionParams &p, uint32_t query_rows, uint32_t key_rows, TensorMaps *m) {
  cudaError_t e;
  if ((e = make_tensor_map_16bit(&m->Q, p.buf[sQ], p.R, p.D, p.batch, query_rows)) != cudaSuccess ||
      (e = make_tensor_map_16bit(&m->dO, p.buf[sdO], p.R, p.D, p.batch, query_rows)) != cudaSuccess)
    return e;
  const uint32_t kv_heads = p.batch / p.group;
  if ((e = make_tensor_map_16bit(&m->K, p.buf[sK], p.C, p.D, kv_heads, key_rows)) != cudaSuccess) return e;
  return make_tensor_map_16bit(&m->V, p.buf[sV], p.C, p.D, kv_heads, key_rows);
}

// The forward kernel of a call's form.  Only the forms compiled above are reachable: the split kernels serve packed and
// paged calls, the FP8 kernels paged ones.
using ForwardKernel = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const FwdArgs);
template <uint32_t DCH, bool kBF16, bool kCausal>
static ForwardKernel forward_kernel(KVLayout layout, bool band, bool split, bool fp8) {
  if (fp8) return band ? fp8_kv_window_forward_wgmma<DCH, kBF16> : fp8_kv_forward_wgmma<DCH, kBF16, kCausal>;
  if (split && layout == KVLayout::kPaged)
    return band ? split_forward_paged_band_wgmma<DCH, kBF16> : split_forward_paged_wgmma<DCH, kBF16, kCausal>;
  if (split) return band ? split_forward_packed_band_wgmma<DCH, kBF16> : split_forward_packed_wgmma<DCH, kBF16, kCausal>;
  if (layout == KVLayout::kPaged) return band ? band_forward_paged_wgmma<DCH, kBF16> : paged_forward_wgmma<DCH, kBF16, kCausal>;
  if (layout == KVLayout::kPacked)
    return band ? band_forward_packed_wgmma<DCH, kBF16> : packed_forward_wgmma<DCH, kBF16, kCausal>;
  return band ? band_forward_wgmma<DCH, kBF16> : attention_forward_wgmma<DCH, kBF16, kCausal>;
}

// A forward call of the form `call` on the grid of `plan`.  Q is read in boxes of kTileM / heads_per_tile rows x
// heads_per_tile heads; K and V as problems of C rows in boxes of BN rows, or (paged) as page pools of C rows, 16-bit
// or FP8, in boxes of min(P, BN) rows.  A packed or paged call runs the split kernels unless the plan has one split and
// one head per tile (FP8: always).  With more than one split the kernel writes partials [split][head][row] into the
// workspace, and merge_splits (fixed) or merge_sequence_splits (packed, paged) merges them into O and L.
template <uint32_t DCH, bool kBF16, bool kCausal>
static cudaError_t launch_forward(const AttentionParams &p, const AttentionCall &call, const WgmmaPlan &plan,
                                  cudaStream_t stream) {
  using Cfg = FwdCfg<DCH>;
  constexpr uint32_t kSmemBytes = Cfg::Smem::kSmemBytes;
  const KVLayout layout = call.pk ? KVLayout::kPaged : (call.seq ? KVLayout::kPacked : KVLayout::kFixed);
  const bool split = layout != KVLayout::kFixed && (call.fp8 || plan.splits > 1 || plan.heads_per_tile > 1);
  const ForwardKernel kernel = forward_kernel<DCH, kBF16, kCausal>(layout, call.band, split, call.fp8);
  const uint32_t hpt = plan.heads_per_tile;
  FwdArgs a{static_cast<float *>(p.buf[sO]), p.buf[sL], p.R, p.C, p.D, p.scale_log2, p.prec[sL], p.causal_offset,
            p.group, SplitArgs{plan.blocks_per_split, plan.splits, p.batch, nullptr, nullptr}, hpt,
            call.seq ? *call.seq : Sequences{}, call.pk ? *call.pk : PagedKV{}, call.band ? *call.band : Band{},
            call.fp8 ? *call.fp8 : Fp8KV{}};
  CUtensorMap mapQ, mapK, mapV;
  cudaError_t e;
  if ((e = prepare(kernel, kSmemBytes)) != cudaSuccess ||
      (e = make_tensor_map_16bit(&mapQ, p.buf[sQ], p.R, p.D, p.batch, Cfg::kTileM / hpt, hpt)) != cudaSuccess)
    return e;
  if (call.pk) {
    const uint32_t box = min(1u << call.pk->page_shift, Cfg::BN);
    auto pool = call.fp8 ? make_tensor_map_page_pool_8bit : make_tensor_map_page_pool;
    if ((e = pool(&mapK, p.buf[sK], p.C, call.pk->kv_heads, p.D, box)) != cudaSuccess ||
        (e = pool(&mapV, p.buf[sV], p.C, call.pk->kv_heads, p.D, box)) != cudaSuccess)
      return e;
  } else if ((e = make_tensor_map_16bit(&mapK, p.buf[sK], p.C, p.D, p.batch / p.group, Cfg::BN)) != cudaSuccess ||
             (e = make_tensor_map_16bit(&mapV, p.buf[sV], p.C, p.D, p.batch / p.group, Cfg::BN)) != cudaSuccess) {
    return e;
  }
  const uint64_t rows_total = static_cast<uint64_t>(p.batch) * p.R;
  if (plan.splits > 1) {
    void *ws = nullptr;
    const size_t o_elems = plan.splits * rows_total * p.D;
    if ((e = workspace_for(current_device(), stream, (o_elems + plan.splits * rows_total) * sizeof(float), &ws)) !=
        cudaSuccess)
      return e;
    a.sp.O_part = static_cast<float *>(ws);
    a.sp.L_part = a.sp.O_part + o_elems;
  }
  kernel<<<plan.grid, Cfg::kThreads, kSmemBytes, stream>>>(mapQ, mapK, mapV, a);
  if ((e = cudaGetLastError()) != cudaSuccess || plan.splits == 1) return e;
  if (layout == KVLayout::kFixed) {
    const uint64_t threads = rows_total * (p.D / 4);
    // (a window can leave a row without a key in a split, or in every split, as causal does)
    auto merge = call.band ? merge_splits<true> : merge_splits<kCausal>;
    merge<<<static_cast<uint32_t>((threads + 127) / 128), 128, 0, stream>>>(a.sp, a.O, a.L, a.l_prec, rows_total, p.D);
  } else {
    const uint64_t threads = static_cast<uint64_t>(call.pk ? call.pk->max_row : call.seq->max_row) * (p.D / 4);
    merge_sequence_splits<<<dim3(static_cast<uint32_t>((threads + 127) / 128), p.batch, plan.grid.z), 128, 0, stream>>>(
        a.sp, a.O, a.L, a.l_prec, p.R, p.D, call.pk ? call.pk->row_offsets : call.seq->row_offsets);
  }
  return cudaGetLastError();
}

// The backward kernel of kernel `type` (dQ or dK/dV) in a call's form
using BackwardKernel = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                                const BwdArgs, const Sequences, const Band);
template <uint32_t DCH, bool kBF16, bool kConvert, bool kCausal>
static BackwardKernel backward_kernel(int type, bool packed, bool band) {
  if (type == MFA_BACKWARD_QUERY) {
    if (band)
      return packed ? band_backward_query_packed_wgmma<DCH, kBF16, kConvert>
                    : band_backward_query_wgmma<DCH, kBF16, kConvert>;
    return packed ? packed_backward_query_wgmma<DCH, kBF16, kConvert, kCausal>
                  : attention_backward_query_wgmma<DCH, kBF16, kConvert, kCausal>;
  }
  if (band)
    return packed ? band_backward_key_value_packed_wgmma<DCH, kBF16, kConvert>
                  : band_backward_key_value_wgmma<DCH, kBF16, kConvert>;
  return packed ? packed_backward_key_value_wgmma<DCH, kBF16, kConvert, kCausal>
                : attention_backward_key_value_wgmma<DCH, kBF16, kConvert, kCausal>;
}

static BwdArgs backward_args(const AttentionParams &p, const WgmmaPlan &plan) {
  BwdArgs a{};
  a.O = static_cast<const float *>(p.buf[sO]);
  a.dO = p.buf[sdO];
  a.L = p.buf[sL];
  a.Dterm = p.buf[sD];
  a.dQ = static_cast<float *>(p.buf[sdQ]);
  a.dK = static_cast<float *>(p.buf[sdK]);
  a.dV = static_cast<float *>(p.buf[sdV]);
  a.blocks_per_split = plan.blocks_per_split;
  a.R = p.R;
  a.C = p.C;
  a.D = p.D;
  a.scale = p.scale;
  a.scale_log2 = p.scale_log2;
  a.l_prec = p.prec[sL];
  a.d_prec = p.prec[sD];
  a.dO_bf16 = p.prec[sdO] == BF16;
  a.delta = p.causal_offset;
  a.group = p.group;
  return a;
}

// Calls f(DCH, kBF16, kConvertDO, kCausal), each as a std::integral_constant, for the kernel instantiation that serves p
template <class F>
static auto dispatch(const AttentionParams &p, bool convert_dO, F f) {
  return with_chunks(p.D, [&](auto dch) {
    auto types = [&](auto causal) {
      if (convert_dO) return f(dch, std::false_type(), std::true_type(), causal);
      if (p.prec[sQ] == BF16) return f(dch, std::true_type(), std::false_type(), causal);
      return f(dch, std::false_type(), std::false_type(), causal);
    };
    return p.causal ? types(std::true_type()) : types(std::false_type());
  });
}

}  // namespace hop

// The plan of fixed-length problems
static WgmmaPlan plan_fixed(int type, uint32_t D, uint32_t R, uint32_t C, uint32_t batch, uint32_t group,
                            uint32_t min_blocks, uint32_t max_splits, bool convert_dO, uint32_t sm_count,
                            const Band *band) {
  WgmmaPlan p{};
  p.heads_per_tile = 1;
  auto geometry = [&](auto cfg) {
    using Cfg = decltype(cfg);
    p.threads = Cfg::kThreads;
    p.smem_bytes = Cfg::Smem::kSmemBytes;
    p.par = Cfg::kPar;
    p.trav = Cfg::kTrav;
  };
  hop::with_chunks(D, [&](auto dch) {
    constexpr uint32_t DCH = decltype(dch)::value;
    if (type == MFA_FORWARD)
      geometry(hop::FwdCfg<DCH>());
    else if (type == MFA_BACKWARD_QUERY)
      geometry(hop::QCfg<DCH>());
    else
      geometry(hop::KVCfg<DCH>());
  });
  const uint32_t padded = (D + 7) / 8 * 8, columns = hop::chunks(D) * 64;
  p.head = columns < padded ? columns : padded;

  const bool key_value = type == MFA_BACKWARD_KEY_VALUE;
  const uint32_t tiles = ((key_value ? C : R) + p.par - 1) / p.par;
  uint32_t total = ((key_value ? R : C) + p.trav - 1) / p.trav;
  if (band) {
    // window: a tile's band covers par + left + right traversal rows, so it meets at most this many blocks (the
    // kernels count each split range from the tile's first visible block)
    const uint64_t width = (static_cast<uint64_t>(p.par) + band->left + band->right + p.trav - 1) / p.trav + 1;
    if (width < total) total = static_cast<uint32_t>(width);
  }
  // CTAs per tile row: one per query head, or for dK/dV one per K/V head (it walks the query heads of its group; the
  // split cuts each head's query blocks the same way)
  const uint32_t heads = key_value ? batch / group : batch;
  if (type == MFA_FORWARD) {
    p.splits = hop::choose_splits(tiles * heads, total, sm_count, min_blocks, max_splits);
    p.blocks_per_split = total / p.splits;
  } else {
    p.blocks_per_split = hop::choose_blocks_per_split(tiles * heads, total, sm_count, min_blocks, max_splits);
    p.splits = (total + p.blocks_per_split - 1) / p.blocks_per_split;
  }
  p.grid = dim3(tiles, heads, p.splits);
  // dK/dV with BF16 dO beside FP16 Q/K/V: a grid of more than one wave converts dO once, in a pass of its own (a
  // smaller one converts each streamed dO tile in shared memory)
  p.convert_dO_first = key_value && convert_dO && static_cast<uint64_t>(tiles) * heads > sm_count;
  // the kernel, + merge_splits / sum_splits when split, + the dO conversion pass
  p.launches = 1 + (p.splits > 1 ? 1 : 0) + (p.convert_dO_first ? 1 : 0);
  return p;
}

// The plan of an unsplit call over `count` packed sequences of at most max_row x max_column
static WgmmaPlan plan_sequences(int type, uint32_t D, uint32_t max_row, uint32_t max_column, uint32_t count,
                                uint32_t batch, uint32_t group, bool convert_dO, uint32_t sm_count) {
  // min_blocks = 0: one traversal range per tile
  WgmmaPlan p = plan_fixed(type, D, max_row, max_column, batch, group, 0, 1, convert_dO, sm_count, nullptr);
  p.grid.z = count;
  p.convert_dO_first = type == MFA_BACKWARD_KEY_VALUE && convert_dO &&
                       static_cast<uint64_t>(p.grid.x) * p.grid.y * count > sm_count;
  p.launches = 1 + (p.convert_dO_first ? 1 : 0);
  return p;
}

// The plan of a split-KV packed or paged forward; every value is host-visible, so launcher, split_plan, grid size and
// launch count agree
static WgmmaPlan plan_split(uint32_t D, uint32_t max_row, uint32_t key_bound, uint32_t count, uint32_t batch,
                            uint32_t group, uint32_t min_blocks, uint32_t max_splits, uint32_t num_splits,
                            uint32_t sm_count, const Band *band) {
  // unsplit, blocks_per_split is the key-block bound of one tile (a window's band width when narrower)
  WgmmaPlan p = plan_fixed(MFA_FORWARD, D, max_row, key_bound, batch, 1, 0, 1, false, sm_count, band);
  // a group's query heads share a tile when an unpacked tile would be partly empty
  p.heads_per_tile = group >= 2 && group <= p.par && max_row < p.par ? group : 1;
  const uint32_t rows = p.par / p.heads_per_tile, tiles = (max_row + rows - 1) / rows;
  const uint64_t items = static_cast<uint64_t>(tiles) * (batch / p.heads_per_tile) * count;
  p.splits = num_splits ? num_splits : hop::choose_key_splits(items, p.blocks_per_split, sm_count, min_blocks, max_splits);
  p.grid = dim3(tiles * p.splits, batch / p.heads_per_tile, count);
  p.launches = 1 + (p.splits > 1 ? 1 : 0);
  return p;
}

WgmmaPlan wgmma_plan(int type, uint32_t D, uint32_t R, uint32_t C, uint32_t batch, uint32_t group, uint32_t min_blocks,
                     uint32_t max_splits, bool convert_dO, const AttentionCall &call, uint32_t sm_count) {
  if (!call.seq && !call.pk)
    return plan_fixed(type, D, R, C, batch, group, min_blocks, max_splits, convert_dO, sm_count, call.band);
  const uint32_t max_row = call.pk ? call.pk->max_row : call.seq->max_row;
  const uint32_t count = call.pk ? call.pk->count : call.seq->count;
  if (call.split) {
    const WgmmaPlan p = plan_split(D, max_row, call.key_bound, count, batch, group, min_blocks, max_splits,
                                   call.num_splits, sm_count, call.band);
    if (p.splits > 1 || p.heads_per_tile > 1) return p;
  }
  // (a paged call's key axis does not enter the grid)
  return plan_sequences(type, D, max_row, call.pk ? 1 : call.seq->max_column, count, batch, group, convert_dO,
                        sm_count);
}

static bool row_major_16bit(const AttentionParams &p) {
  for (int s = 0; s < kSlots; ++s)
    if (p.transposed[s]) return false;
  return (p.prec[sQ] == FP16 || p.prec[sQ] == BF16) && p.prec[sK] == p.prec[sQ] && p.prec[sV] == p.prec[sQ] &&
         p.D % 8 == 0 && p.D <= kWgmmaMaxHead;
}

static cudaError_t check_backward(const AttentionParams &p) {
  const bool dO_ok = p.prec[sdO] == p.prec[sQ] || (p.prec[sQ] == FP16 && p.prec[sdO] == BF16);
  if (row_major_16bit(p) && dO_ok && p.prec[sO] == FP32 && p.prec[sdQ] == FP32 && p.prec[sdK] == FP32 &&
      p.prec[sdV] == FP32)
    return cudaSuccess;
  set_launch_detail("descriptor is outside the wgmma backward kernels' domain");
  return cudaErrorInvalidValue;
}

// A backward call of kernel `type` in the form `call` on the grid of its plan.  dK/dV with BF16 dO beside FP16 Q/K/V on
// a grid of more than one wave: a pass of its own converts dO to FP16 first.  Split: each split writes partial sums of
// the outputs (dQ; or dV and dK, per K/V head) to the workspace, [split][output][elems], and sum_splits adds them into
// the outputs.
static cudaError_t launch_backward(int type, const AttentionParams &p, const AttentionCall &call, cudaStream_t stream) {
  if (cudaError_t e = check_backward(p)) return e;
  const bool convert = p.prec[sdO] != p.prec[sQ], key_value = type == MFA_BACKWARD_KEY_VALUE;
  const WgmmaPlan plan = wgmma_plan(type, p.D, p.R, p.C, p.batch, p.group, p.split_min_blocks, p.split_max, convert,
                                    call, device_sm_count(current_device()));
  AttentionParams q = p;
  cudaError_t e;
  if (plan.convert_dO_first) {
    const uint64_t elements = static_cast<uint64_t>(p.batch) * p.R * p.D;
    void *converted = nullptr;
    if ((e = workspace_for(current_device(), stream, elements * 2, &converted, /*slot=*/2)) != cudaSuccess ||
        (e = launch_bf16_to_f16(p.buf[sdO], converted, elements, stream)) != cudaSuccess)
      return e;
    q.buf[sdO] = converted;
    q.prec[sdO] = q.prec[sQ];
  }
  const hop::BackwardKernel kernel =
      hop::dispatch(q, convert && !plan.convert_dO_first, [&](auto dch, auto bf16, auto cvt, auto causal) {
        return hop::backward_kernel<decltype(dch)::value, decltype(bf16)::value, decltype(cvt)::value,
                                    decltype(causal)::value>(type, call.seq, call.band);
      });
  hop::TensorMaps m;
  if ((e = hop::prepare(kernel, plan.smem_bytes)) != cudaSuccess ||
      (e = hop::make_maps(q, key_value ? plan.trav : plan.par, key_value ? plan.par : plan.trav, &m)) != cudaSuccess)
    return e;
  hop::BwdArgs a = hop::backward_args(q, plan);
  const uint32_t outputs = key_value ? 2 : 1;
  const size_t elems = key_value ? static_cast<size_t>(q.batch / q.group) * q.C * q.D
                                 : static_cast<size_t>(q.batch) * q.R * q.D;
  float *const out0 = key_value ? a.dV : a.dQ, *const out1 = key_value ? a.dK : nullptr;
  float *part = nullptr;
  if (plan.splits > 1) {
    void *ws = nullptr;
    const size_t bytes = plan.splits * outputs * elems * sizeof(float);
    if ((e = workspace_for(current_device(), stream, bytes, &ws)) != cudaSuccess) return e;
    part = static_cast<float *>(ws);
    a.split_stride = outputs * elems;
    (key_value ? a.dV : a.dQ) = part;
    if (key_value) a.dK = part + elems;
  }
  kernel<<<plan.grid, plan.threads, plan.smem_bytes, stream>>>(m.Q, m.dO, m.K, m.V, a, call.seq ? *call.seq : Sequences{},
                                                               call.band ? *call.band : Band{});
  if ((e = cudaGetLastError()) != cudaSuccess || plan.splits == 1) return e;
  const size_t quads = elems / 4;  // D % 8 == 0
  hop::sum_splits<<<dim3(static_cast<uint32_t>((quads + 255) / 256), outputs), 256, 0, stream>>>(
      reinterpret_cast<const float4 *>(part), reinterpret_cast<float4 *>(out0), reinterpret_cast<float4 *>(out1), quads,
      a.split_stride / 4, plan.splits);
  return cudaGetLastError();
}

cudaError_t launch_wgmma(int type, const AttentionParams &p, const AttentionCall &call, cudaStream_t stream) {
  if (type != MFA_FORWARD) return launch_backward(type, p, call, stream);
  if (!row_major_16bit(p) || p.prec[sO] != FP32 || (call.fp8 && p.D % 16 != 0)) {
    set_launch_detail(call.fp8 ? "descriptor is outside the FP8 K/V forward kernels' domain"
                               : "descriptor is outside the wgmma forward kernel's domain");
    return cudaErrorInvalidValue;
  }
  const WgmmaPlan plan = wgmma_plan(MFA_FORWARD, p.D, p.R, p.C, p.batch, p.group, p.split_min_blocks, p.split_max,
                                    false, call, device_sm_count(current_device()));
  return hop::dispatch(p, false, [&](auto dch, auto bf16, auto, auto causal) {
    return hop::launch_forward<decltype(dch)::value, decltype(bf16)::value, decltype(causal)::value>(p, call, plan,
                                                                                                      stream);
  });
}

}  // namespace mfa
