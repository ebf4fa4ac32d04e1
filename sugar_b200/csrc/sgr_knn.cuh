// sgr_knn.cuh -- the uniform cell grid of sgr_knn.cu, shared with the density grid of sgr_mcubes.cu.
#pragma once
#include "sgr_internal.cuh"

namespace sgr {

struct KnnGrid {
    float lo[3];
    float inv_h;  // cells per unit length (cubic cells)
    float h;      // cell edge
    int n[3];     // cells per axis, n[0] * n[1] * n[2] <= the budget N^3
};

constexpr int KNN_MAXK = 64;

#ifdef __CUDACC__
__device__ __forceinline__ int cell_coord(float v, float lo, float inv_h, int n)
{
    const int c = (int)floorf((v - lo) * inv_h);
    return min(max(c, 0), n - 1);
}
#endif

// The reference points sorted by cell: cell c holds sorted[starts[c] .. starts[c + 1]) (the last cell ends at P), each
// entry (x, y, z, index bits).  Everything stays on the device.
struct KnnCells {
    const KnnGrid *grid;
    const uint32_t *starts;
    const float4 *sorted;
};

// knn_build_cells' workspace
struct KnnCellsScratch {
    int *bbox;
    KnnGrid *grid;
    uint32_t *cell_of, *starts, *cursor, *bsums;
    float4 *sorted;
};
KnnCellsScratch knn_cells_scratch(Layout &l, int P);
int knn_build_cells(int P, const float *points, const KnnCellsScratch &ws, cudaStream_t st, KnnCells *out);

// The block sums exclusive_scan_u32 needs for n counts.
static inline size_t scan_block_sums(size_t n) { return (n + 4095) / 4096 + 1; }

// Exclusive scan of n uint32 counts into starts (counts == starts is allowed), written to cursor as well;
// block_sums holds scan_block_sums(n) entries.  Three launches under `kind`.
void exclusive_scan_u32(int kind, int n, const uint32_t *counts, uint32_t *starts, uint32_t *block_sums,
                        uint32_t *cursor, cudaStream_t st);

}  // namespace sgr
