// Host-side TMA tensor-map construction (cuTensorMapEncodeTiled resolved through the runtime's
// driver entry point, so the library needs no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mfa {

// Row-major [batch][seq][D] matrix of 16-bit elements, tiled as boxes of 64 (D) x box_rows (seq) x box_depth
// (problems), 128-byte swizzle, out-of-bounds elements read as zero (the analogue of the reference's zero-padded
// async copies, GEMMHeaders.swift:111-114).  A box of depth n lands as n [box_rows][64] tiles one after another, which
// the swizzle (a function of the shared-memory address) lays out as one [n * box_rows][64] tile.
cudaError_t make_tensor_map_16bit(CUtensorMap *map, const void *base, uint32_t seq, uint32_t D, uint32_t batch,
                                  uint32_t box_rows, uint32_t box_depth = 1);

// Page pool [rows][heads][D] of 16-bit elements (a paged K/V cache): dims {D, heads, rows}, boxes of 64 (D) x 1 (head)
// x box_rows (rows), loaded at (column, head, row) into the same [box_rows][64] 128-byte-swizzled tile as above.
cudaError_t make_tensor_map_page_pool(CUtensorMap *map, const void *base, uint32_t rows, uint32_t heads, uint32_t D,
                                      uint32_t box_rows);

// The same pool of 1-byte elements (FP8 K/V): boxes of 64 (D) x 1 (head) x box_rows bytes, unswizzled, landing as a
// dense [box_rows][64]-byte tile.  D must be a multiple of 16 (16-byte row pitch).
cudaError_t make_tensor_map_page_pool_8bit(CUtensorMap *map, const void *base, uint32_t rows, uint32_t heads,
                                           uint32_t D, uint32_t box_rows);

void set_launch_detail(const char *fmt, ...);

}  // namespace mfa
