// sgr_knn.cu -- exact K-nearest-neighbour search on a uniform grid (sm_90a).
//
// Replaces pytorch3d.ops.knn_points as SuGaR uses it (pytorch3d 0.7.4 is not part of the reference
// tree; call sites: sugar_scene/sugar_model.py:1013-1030 `reset_neighbors` = knn_points(points,
// points, K=16) every 500 iterations, and :1335-1343 `get_gaussians_closest_to_samples`).
// Semantics kept: exact K nearest by squared Euclidean distance, results ordered by increasing
// distance, int64 indices, a point is its own neighbour 0 when queries == points.  Ties may be
// returned in a different order than pytorch3d (which does not define one).
//
// Method: counting sort of the reference points into a grid of CUBIC cells over their bounding box
// (per-axis cell counts nx x ny x nz <= N^3, the edge chosen on the device so that the cell count
// approaches the budget: a flat or elongated cloud gets a 2-D / 1-D grid instead of N layers of
// empty or paper-thin cells), then one thread per query walks Chebyshev shells of cells around its
// own cell with a K-entry insertion list in local memory; after shell r every unvisited point is
// farther than r * (cell edge), which bounds the search exactly.  Everything (bounding box, cell
// size) stays on the device: no host synchronisation.
#include <math.h>

#include "sgr_knn.cuh"

namespace sgr {

__device__ __forceinline__ int float_flip(float f)
{  // order-preserving float -> int map for atomicMin/Max
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float float_unflip(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// bb: int[6] flipped min / max per axis, then (8-byte aligned) double[6] sum / sum of squares per axis
__global__ void knn_bbox_init_kernel(int *bb)
{
    if (threadIdx.x < 3) bb[threadIdx.x] = 0x7fffffff;
    else if (threadIdx.x < 6) bb[threadIdx.x] = (int)0x80000000;
    else if (threadIdx.x < 12) ((double *)(bb + 8))[threadIdx.x - 6] = 0.0;
}

__global__ void __launch_bounds__(256) knn_bbox_kernel(int P, const float *__restrict__ pts, int *bb)
{
    float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
    double s1[3] = {0, 0, 0}, s2[3] = {0, 0, 0};
    for (int i = blockIdx.x * 256 + threadIdx.x; i < P; i += gridDim.x * 256) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float v = pts[3 * i + a];
            mn[a] = fminf(mn[a], v);
            mx[a] = fmaxf(mx[a], v);
            s1[a] += (double)v;
            s2[a] += (double)v * (double)v;
        }
    }
    double *mom = (double *)(bb + 8);
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const int lo = __reduce_min_sync(0xffffffffu, float_flip(mn[a]));
        const int hi = __reduce_max_sync(0xffffffffu, float_flip(mx[a]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s1[a] += __shfl_xor_sync(0xffffffffu, s1[a], o);
            s2[a] += __shfl_xor_sync(0xffffffffu, s2[a], o);
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&bb[a], lo);
            atomicMax(&bb[3 + a], hi);
            atomicAdd(&mom[a], s1[a]);
            atomicAdd(&mom[3 + a], s2[a]);
        }
    }
}

// The grid covers the bounding box clipped to mean +- 4 sigma per axis: a few far outliers (floaters) would
// otherwise stretch the box and leave the bulk of the cloud in a handful of cells.  Points outside the clipped
// box are clamped into the border cells, which keeps the shell bound valid (they are only farther away than
// their cell suggests).
__global__ void knn_grid_setup_kernel(const int *bb, int n, int P, KnnGrid *g)
{
    if (threadIdx.x != 0) return;
    const double *mom = (const double *)(bb + 8);
    float ext[3], emax = 0.f;
    for (int a = 0; a < 3; a++) {
        float lo = float_unflip(bb[a]), hi = float_unflip(bb[3 + a]);
        const double mean = mom[a] / (double)P, var = fmax(mom[3 + a] / (double)P - mean * mean, 0.0);
        const float sd = (float)sqrt(var), m = (float)mean;
        if (sd > 0.f) {
            lo = fmaxf(lo, m - 4.0f * sd);
            hi = fminf(hi, m + 4.0f * sd);
        }
        ext[a] = hi - lo;
        if (!(ext[a] > 0.f)) ext[a] = 0.f;
        emax = fmaxf(emax, ext[a]);
        g->lo[a] = lo;
    }
    if (!(emax > 1e-30f)) emax = 1e-30f;  // all points coincide: one cell
    // smallest cubic edge whose grid fits the budget of n^3 cells: bisection on the edge length
    // (cells(h) is monotone; h never drops below longest extent / 8 n)
    const double budget = (double)n * n * n;
    auto cells = [&](float h, int *c) {
        double prod = 1.0;
        for (int a = 0; a < 3; a++) {
            const float k = floorf(ext[a] / h) + 1.0f;
            c[a] = (int)fminf(k, 1.0e6f);
            prod *= (double)c[a];
        }
        return prod;
    };
    float h_hi = emax * 1.0001f, h_lo = emax / (8.0f * (float)n);
    int c[3];
    for (int it = 0; it < 40; it++) {
        const float mid = 0.5f * (h_lo + h_hi);
        if (cells(mid, c) <= budget) h_hi = mid;
        else h_lo = mid;
    }
    cells(h_hi, c);
    g->h = h_hi;
    g->inv_h = 1.0f / h_hi;
    for (int a = 0; a < 3; a++) g->n[a] = c[a];
}

__global__ void __launch_bounds__(256) knn_count_kernel(int P, const float *__restrict__ pts, const KnnGrid *__restrict__ gp,
                                                        uint32_t *__restrict__ cell_of, uint32_t *__restrict__ counts)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    const KnnGrid g = *gp;
    const int cx = cell_coord(pts[3 * i], g.lo[0], g.inv_h, g.n[0]);
    const int cy = cell_coord(pts[3 * i + 1], g.lo[1], g.inv_h, g.n[1]);
    const int cz = cell_coord(pts[3 * i + 2], g.lo[2], g.inv_h, g.n[2]);
    const uint32_t c = ((uint32_t)cz * g.n[1] + cy) * g.n[0] + cx;
    cell_of[i] = c;
    atomicAdd(&counts[c], 1u);
}

// three-kernel exclusive scan over the cell counts (block = 1024 threads x 4 cells); in place is safe: a thread loads
// its four counts before the block barrier and stores their offsets after it
__global__ void __launch_bounds__(1024) knn_scan_blocks_kernel(int ncell, const uint32_t *__restrict__ counts,
                                                               uint32_t *__restrict__ starts, uint32_t *__restrict__ block_sums)
{
    __shared__ uint32_t s_w[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int i0 = (blockIdx.x * 1024 + tid) * 4;
    uint32_t v[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        v[k] = (i0 + k < ncell) ? counts[i0 + k] : 0u;
        sum += v[k];
    }
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = s_w[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        s_w[lane] = wi - w;
        if (lane == 31) block_sums[blockIdx.x] = wi;
    }
    __syncthreads();
    uint32_t ex = s_w[wid] + inc - sum;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (i0 + k < ncell) starts[i0 + k] = ex;
        ex += v[k];
    }
}

__global__ void __launch_bounds__(1024) knn_scan_sums_kernel(int nblocks, uint32_t *block_sums)
{
    // single CTA, serial over chunks of 1024 (nblocks <= 4096 for 2^24 cells)
    __shared__ uint32_t s_w[32];
    __shared__ uint32_t s_carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        const uint32_t v = (base + tid < nblocks) ? block_sums[base + tid] : 0u;
        uint32_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = s_w[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            s_w[lane] = wi - w;
        }
        __syncthreads();
        const uint32_t ex = s_carry + s_w[wid] + inc - v;
        if (base + tid < nblocks) block_sums[base + tid] = ex;
        __syncthreads();
        if (tid == 1023) s_carry = ex + v;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(1024) knn_scan_add_kernel(int ncell, uint32_t *__restrict__ starts,
                                                            const uint32_t *__restrict__ block_sums,
                                                            uint32_t *__restrict__ cursor)
{
    const int i0 = (blockIdx.x * 1024 + threadIdx.x) * 4;
    const uint32_t add = block_sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (i0 + k < ncell) {
            const uint32_t s = starts[i0 + k] + add;
            starts[i0 + k] = s;
            cursor[i0 + k] = s;
        }
}

__global__ void __launch_bounds__(256) knn_scatter_kernel(int P, const float *__restrict__ pts,
                                                          const uint32_t *__restrict__ cell_of, uint32_t *__restrict__ cursor,
                                                          float4 *__restrict__ sorted)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    const uint32_t slot = atomicAdd(&cursor[cell_of[i]], 1u);
    sorted[slot] = make_float4(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], __int_as_float(i));
}

__global__ void __launch_bounds__(128) knn_query_kernel(int Q, int K, int P, const float *__restrict__ qs,
                                                        const KnnGrid *__restrict__ gp, const uint32_t *__restrict__ starts,
                                                        const float4 *__restrict__ sorted, int64_t *__restrict__ idx_out,
                                                        float *__restrict__ d2_out)
{
    const int q = blockIdx.x * 128 + threadIdx.x;
    if (q >= Q) return;
    const KnnGrid g = *gp;
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const uint32_t ncell = (uint32_t)nx * ny * nz;
    const float qx = qs[3 * q], qy = qs[3 * q + 1], qz = qs[3 * q + 2];
    const int cx = cell_coord(qx, g.lo[0], g.inv_h, nx), cy = cell_coord(qy, g.lo[1], g.inv_h, ny),
              cz = cell_coord(qz, g.lo[2], g.inv_h, nz);
    const int rmax = max(nx, max(ny, nz));
    // a query outside the bounding box is first clamped into the border cell; the shell bound below
    // then needs the distance from the query to that cell, which only makes the bound smaller
    float best_d[KNN_MAXK];
    int best_i[KNN_MAXK];
    int have = 0;
    float kth = 3.0e38f;
    const uint32_t total = (uint32_t)P;
    for (int r = 0; r < rmax; r++) {
        const int z0 = max(cz - r, 0), z1 = min(cz + r, nz - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, ny - 1);
        const int x0 = max(cx - r, 0), x1 = min(cx + r, nx - 1);
        for (int z = z0; z <= z1; z++) {
            const bool zface = (z == cz - r) || (z == cz + r);
            for (int y = y0; y <= y1; y++) {
                const bool yface = (y == cy - r) || (y == cy + r);
                // on a z- or y-face the whole x-run belongs to the shell; otherwise only its two ends
                const int step = (zface || yface || r == 0) ? 1 : max(1, 2 * r);
                for (int x = cx - r; x <= cx + r; x += step) {
                    if (x < x0 || x > x1) continue;
                    const uint32_t c = ((uint32_t)z * ny + y) * nx + x;
                    const uint32_t s = starts[c];
                    const uint32_t e = (c + 1 < ncell) ? starts[c + 1] : total;
                    for (uint32_t k = s; k < e; k++) {
                        const float4 p = __ldg(sorted + k);
                        const float dx = p.x - qx, dy = p.y - qy, dz = p.z - qz;
                        const float d2 = dx * dx + dy * dy + dz * dz;
                        if (have < K || d2 < kth) {
                            int j = have < K ? have : K - 1;  // insertion position search from the back
                            while (j > 0 && best_d[j - 1] > d2) {
                                best_d[j] = best_d[j - 1];
                                best_i[j] = best_i[j - 1];
                                j--;
                            }
                            best_d[j] = d2;
                            best_i[j] = __float_as_int(p.w);
                            if (have < K) have++;
                            if (have == K) kth = best_d[K - 1];
                        }
                    }
                }
            }
        }
        // every unvisited point lies beyond shell r: farther than r cell edges from the query's cell, hence
        // from the query if it is inside the box; outside the box the query is even farther from them
        const float bound = (float)r * g.h;
        if (have == K && kth <= bound * bound) break;
    }
    for (int j = 0; j < K; j++) {
        idx_out[(size_t)q * K + j] = j < have ? (int64_t)best_i[j] : (int64_t)-1;
        d2_out[(size_t)q * K + j] = j < have ? best_d[j] : 0.0f;
    }
}

static int knn_axis_cells(int P)
{
    // about 4 points per cell on a volume-filling cloud; surface-like clouds leave most cells empty,
    // which only costs the (cheap) empty-cell visits.  Capped at 256^3 = 16.7M cells.
    int n = (int)ceil(cbrt((double)P / 4.0));
    if (n < 1) n = 1;
    if (n > 256) n = 256;
    return n;
}

size_t knn_cells_bytes(int P)
{
    const size_t n = (size_t)knn_axis_cells(P < 1 ? 1 : P), ncell = n * n * n;
    const size_t nblocks = (ncell + 4095) / 4096;
    return align_up(64) + align_up(sizeof(KnnGrid)) + align_up((size_t)P * 4) + 2 * align_up((ncell + 1) * 4) +
           align_up((nblocks + 1) * 4) + align_up((size_t)P * 16) + SGR_ALIGN;
}

void exclusive_scan_u32(int kind, int n, const uint32_t *counts, uint32_t *starts, uint32_t *block_sums,
                        uint32_t *cursor, cudaStream_t st)
{
    const int nblocks = (int)(((size_t)n + 4095) / 4096);
    SGR_LAUNCH(kind, st, knn_scan_blocks_kernel<<<(unsigned)nblocks, 1024, 0, st>>>(n, counts, starts, block_sums));
    SGR_LAUNCH(kind, st, knn_scan_sums_kernel<<<1, 1024, 0, st>>>(nblocks, block_sums));
    SGR_LAUNCH(kind, st, knn_scan_add_kernel<<<(unsigned)nblocks, 1024, 0, st>>>(n, starts, block_sums, cursor));
}

int knn_build_cells(int P, const float *points, void *workspace, cudaStream_t st, KnnCells *out)
{
    const int n = knn_axis_cells(P);
    const size_t ncell = (size_t)n * n * n, nblocks = (ncell + 4095) / 4096;
    char *p = (char *)align_up((size_t)workspace);
    int *bb = (int *)p; p += align_up(64);
    KnnGrid *grid = (KnnGrid *)p; p += align_up(sizeof(KnnGrid));
    uint32_t *cell_of = (uint32_t *)p; p += align_up((size_t)P * 4);
    uint32_t *starts = (uint32_t *)p; p += align_up((ncell + 1) * 4);
    uint32_t *cursor = (uint32_t *)p; p += align_up((ncell + 1) * 4);
    uint32_t *bsums = (uint32_t *)p; p += align_up((nblocks + 1) * 4);
    float4 *sorted = (float4 *)p;
    SGR_LAUNCH(K_KNN, st, knn_bbox_init_kernel<<<1, 32, 0, st>>>(bb));
    SGR_LAUNCH(K_KNN, st, knn_bbox_kernel<<<device_sm_count() * 4, 256, 0, st>>>(P, points, bb));
    SGR_LAUNCH(K_KNN, st, knn_grid_setup_kernel<<<1, 32, 0, st>>>(bb, n, P, grid));
    SGR_CUDA(cudaMemsetAsync(cursor, 0, ncell * 4, st));  // cursor doubles as the count array first
    SGR_LAUNCH(K_KNN, st, knn_count_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, points, grid, cell_of, cursor));
    exclusive_scan_u32(K_KNN, (int)ncell, cursor, starts, bsums, cursor, st);
    SGR_LAUNCH(K_KNN, st, knn_scatter_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, points, cell_of, cursor, sorted));
    out->grid = grid;
    out->starts = starts;
    out->sorted = sorted;
    return SGR_OK;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

size_t sgr_knn_workspace_bytes(int32_t P) { return knn_cells_bytes(P); }

int sgr_knn(int32_t P, const float *points, int32_t Q, const float *queries, int32_t K, int64_t *idx, float *dist2,
            void *workspace, void *stream)
{
    if (P <= 0 || Q < 0 || K <= 0 || K > KNN_MAXK || K > P || !points || (Q > 0 && (!queries || !idx || !dist2)) ||
        !workspace) {
        set_error("sgr_knn: need 0 < K <= min(P, %d), non-null pointers (P=%d Q=%d K=%d)", KNN_MAXK, P, Q, K);
        return SGR_EINVAL;
    }
    if (Q == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    KnnCells cells;
    int rc = knn_build_cells(P, points, workspace, st, &cells);
    if (rc) return rc;
    SGR_LAUNCH(K_KNN_QUERY, st,
               knn_query_kernel<<<(Q + 127) / 128, 128, 0, st>>>(Q, K, P, queries, cells.grid, cells.starts,
                                                                 cells.sorted, idx, dist2));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
