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

// The squared distance of a pair as the walks compute it: every step rounded on its own, ((dx dx + dy dy) + dz dz) with
// d = p - q and no contraction, so that float32 tensor ops (one op per rounding) reproduce it to the bit.
__device__ __forceinline__ float knn_dist2(float px, float py, float pz, float qx, float qy, float qz)
{
    const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// The walks' order: by distance, equal distances by index.  The K nearest under it do not depend on the order in which
// the walk meets the points (the cells' order comes from atomics), so a cloud with duplicates has one answer.
__device__ __forceinline__ bool knn_before(float d2, int id, float other_d2, int other_id)
{
    return d2 < other_d2 || (d2 == other_d2 && id < other_id);
}

// After shell r every unvisited point is more than (r - KNN_SHELL_MARGIN) cell edges from the query.  The margin covers
// cell_coord's rounding: an axis has at most 8 n + 1 <= 2049 cells (knn_grid_setup_kernel), and (v - lo) * inv_h is off
// by at most about 3 * 2^-24 * 2049 ~ 3.7e-4 cells, so a point and a query filed one cell over each are together less
// than 1e-3 edges out.  A walk stops once the K-th distance is strictly below this radius squared: an unvisited point at
// exactly that distance could still come first by index.
constexpr float KNN_SHELL_MARGIN = 1e-3f;
__device__ __forceinline__ float knn_shell_radius(int r, float h) { return fmaxf((float)r - KNN_SHELL_MARGIN, 0.0f) * h; }
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

}  // namespace sgr
