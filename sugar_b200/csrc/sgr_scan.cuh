// sgr_scan.cuh -- the device-wide exclusive scan of sgr_scan.cu.
#pragma once
#include "sgr_internal.cuh"

namespace sgr {

// The block sums exclusive_scan needs for n counts.
static inline size_t scan_block_sums(size_t n) { return (n + 4095) / 4096 + 1; }

// Exclusive scan of n uint32 counts into starts, written to cursor as well (cursor == starts writes once);
// block_sums holds scan_block_sums(n) entries.  T is the offset type: uint32_t (counts may alias starts or cursor)
// or unsigned long long.  A caller that needs
// the grand total appends a zero count and reads starts[n - 1].  Three launches under `kind`; integer sums, so the
// result does not depend on the blocking.
template <typename T>
void exclusive_scan(int kind, size_t n, const uint32_t *counts, T *starts, T *block_sums, T *cursor, cudaStream_t st);

}  // namespace sgr
