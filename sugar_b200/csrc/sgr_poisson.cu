// sgr_poisson.cu -- screened-Poisson surface reconstruction on a dense grid (sm_90a): the splat of oriented samples
// onto trilinear hats and a geometric-multigrid solve of the 7-point screened system.  sugar_b200/poisson.py states
// the discrete problem; oracle/poisson_oracle.py restates it in float64.
//
// Grid: N = 2^depth nodes per axis, C order (x slowest, z fastest), node (i, j, k) at grid units (i, j, k).  A sample's
// grid coordinates are g = (p - o) * inv_h - 0.5 in float32, each operation rounded once (the oracle repeats them).
//
// Splat: every sample goes to the bin of its hat support's lower corner node L = clamp(floor(g), 0, N - 2).  Bin counts
// (integer atomics) and sgr_knn.cu's exclusive scan give each bin's start; a stable LSD radix sort of the records by
// bin key (8 bits per pass, tiles of 256 keys, one exclusive scan of the digit-major tile histograms per pass) puts
// each bin's samples in sample order at a cost linear in n whatever the bins' sizes.  A node then gathers from its 8
// neighbouring bins in increasing bin index, each in sample order, and writes its value once: no float atomics, so
// every grid is bit-identical from run to run.
//
// Solve: V(2,2) cycles.  Red-black Gauss-Seidel on sum_{j in N6(i)} c (u_i - u_j) + q_i u_i = b_i with c = 2^level
// (a trilinear stiffness scales with the spacing) and missing neighbours dropped (zero flux); the restriction sums the
// residuals of a coarse node's 8 children, the prolongation is cell-centred trilinear (weights 3/4, 1/4 per axis,
// constant beyond the faces); coarse q sums the 8 children's q.  The 4^3 level is smoothed to convergence by one CTA.
// Norms and sums are double-precision block reductions over a fixed grid of POI_RED_BLOCKS blocks, summed in a fixed
// order; the host reads one scalar per call.
#include <math.h>

#include "sgr_reduce.cuh"
#include "sgr_scan.cuh"

namespace sgr {

constexpr int POI_RED_BLOCKS = 1024;  // partial sums of every reduction (the caller's `partial` holds this many doubles)
constexpr int POI_COARSEST_SWEEPS = 64;

static inline unsigned blocks_for(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

__device__ __forceinline__ float grid_coord(float p, float o, float inv_h)
{
    return __fsub_rn(__fmul_rn(__fsub_rn(p, o), inv_h), 0.5f);
}

__device__ __forceinline__ int lower_node(float g, int N) { return min(max((int)floorf(g), 0), N - 2); }

__device__ __forceinline__ uint32_t bin_of(const float *__restrict__ p, float ox, float oy, float oz, float inv_h, int N)
{
    const int x = lower_node(grid_coord(p[0], ox, inv_h), N);
    const int y = lower_node(grid_coord(p[1], oy, inv_h), N);
    const int z = lower_node(grid_coord(p[2], oz, inv_h), N);
    return ((uint32_t)x * N + y) * N + z;
}

// the bin key of every sample, its record in sample order, and the bins' counts (integer atomics: order-free)
__global__ void __launch_bounds__(256) poi_key_kernel(int n, const float *__restrict__ pts, float ox, float oy, float oz,
                                                      float inv_h, int N, uint32_t *__restrict__ keys,
                                                      float4 *__restrict__ rec, uint32_t *__restrict__ counts)
{
    const int s = blockIdx.x * 256 + threadIdx.x;
    if (s >= n) return;
    const float *p = pts + 3 * (size_t)s;
    const uint32_t b = bin_of(p, ox, oy, oz, inv_h, N);
    keys[s] = b;
    rec[s] = make_float4(grid_coord(p[0], ox, inv_h), grid_coord(p[1], oy, inv_h), grid_coord(p[2], oz, inv_h),
                         __int_as_float(s));
    atomicAdd(&counts[b], 1u);
}

// Stable LSD radix sort of the records by bin key, 8 bits per pass: a tile is 256 consecutive keys (one CTA).
// hist: the tile's digit counts, stored digit-major so that one exclusive scan gives every (digit, tile) offset.
constexpr int POI_RADIX_TILE = 256;

__global__ void __launch_bounds__(POI_RADIX_TILE) poi_radix_hist_kernel(int n, const uint32_t *__restrict__ keys, int shift,
                                                                         int ntiles, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t h[256];
    const int t = threadIdx.x, i = blockIdx.x * POI_RADIX_TILE + t;
    h[t] = 0;
    __syncthreads();
    if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255u], 1u);
    __syncthreads();
    hist[(size_t)t * ntiles + blockIdx.x] = h[t];
}

// scatter: a key's slot is its (digit, tile) offset + the same-digit keys of earlier warps of the tile + those of
// earlier lanes of its warp, so equal digits keep their order and the sort is stable
__global__ void __launch_bounds__(POI_RADIX_TILE) poi_radix_scatter_kernel(int n, const uint32_t *__restrict__ keys_in,
                                                                            const float4 *__restrict__ rec_in, int shift,
                                                                            int ntiles, const uint32_t *__restrict__ offs,
                                                                            uint32_t *__restrict__ keys_out,
                                                                            float4 *__restrict__ rec_out)
{
    constexpr int W = POI_RADIX_TILE / 32;
    __shared__ uint32_t wc[W][256];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, i = blockIdx.x * POI_RADIX_TILE + t;
    for (int k = t; k < W * 256; k += POI_RADIX_TILE) (&wc[0][0])[k] = 0;
    __syncthreads();
    const bool valid = i < n;
    const uint32_t key = valid ? keys_in[i] : 0u;
    const uint32_t digit = (key >> shift) & 255u;
    const unsigned same = __match_any_sync(0xffffffffu, valid ? digit : 256u + lane);
    const unsigned rank = __popc(same & ((1u << lane) - 1u));
    if (valid && rank == 0) wc[warp][digit] = __popc(same);
    __syncthreads();
    if (!valid) return;
    uint32_t slot = offs[(size_t)digit * ntiles + blockIdx.x] + rank;
    for (int w = 0; w < warp; w++) slot += wc[w][digit];
    keys_out[slot] = key;
    rec_out[slot] = rec_in[i];
}

// the number of occupied bins: the first key of each run of the sorted keys
__global__ void __launch_bounds__(256) poi_occupied_kernel(int n, const uint32_t *__restrict__ keys,
                                                           uint32_t *__restrict__ occupied)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    const bool first = i < n && (i == 0 || keys[i] != keys[i - 1]);
    const unsigned m = __ballot_sync(0xffffffffu, first);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(occupied, (uint32_t)__popc(m));
}

// bin b holds binned[starts[b] .. starts[b + 1]), the last bin ending at n
__device__ __forceinline__ uint32_t bin_end(const uint32_t *__restrict__ starts, size_t b, size_t nbins, uint32_t n)
{
    return b + 1 < nbins ? starts[b + 1] : n;
}

enum PoiSplat { POI_SYSTEM = 0, POI_WEIGHT = 1, POI_ATTRIBUTE = 2 };

// One thread per node: the 8 bins whose cube has this node as a corner, in increasing bin index, each in sample order.
//   POI_SYSTEM:    out0 = -area * sum n . grad phi,  out1 = alpha * area * sum phi   (attr = normals [n,3])
//   POI_WEIGHT:    out0 = sum phi
//   POI_ATTRIBUTE: out0 = sum phi * attr[s, channel]                                  (attr [n,3])
template <int MODE>
__global__ void __launch_bounds__(256) poi_splat_kernel(int N, uint32_t n, const uint32_t *__restrict__ starts,
                                                        const float4 *__restrict__ binned, const float *__restrict__ attr,
                                                        int channel, float area, float alpha, float *__restrict__ out0,
                                                        float *__restrict__ out1)
{
    const size_t node = (size_t)blockIdx.x * 256 + threadIdx.x;
    const size_t NN = (size_t)N * N;
    if (node >= NN * N) return;
    const int i = (int)(node / NN), j = (int)(node / N % N), k = (int)(node % N);
    float acc0 = 0.0f, acc1 = 0.0f;
    for (int dx = -1; dx <= 0; dx++) {
        const int lx = i + dx;
        if (lx < 0 || lx > N - 2) continue;
        for (int dy = -1; dy <= 0; dy++) {
            const int ly = j + dy;
            if (ly < 0 || ly > N - 2) continue;
            for (int dz = -1; dz <= 0; dz++) {
                const int lz = k + dz;
                if (lz < 0 || lz > N - 2) continue;
                const size_t b = ((size_t)lx * N + ly) * N + lz;
                const uint32_t e = bin_end(starts, b, NN * N, n);
                for (uint32_t s = starts[b]; s < e; s++) {
                    const float4 r = binned[s];
                    // this node is the bin's lower corner along an axis when d = 0: weight 1 - t, slope -1
                    const float tx = __fsub_rn(r.x, (float)lx), ty = __fsub_rn(r.y, (float)ly), tz = __fsub_rn(r.z, (float)lz);
                    const float wx = dx ? tx : __fsub_rn(1.0f, tx);
                    const float wy = dy ? ty : __fsub_rn(1.0f, ty);
                    const float wz = dz ? tz : __fsub_rn(1.0f, tz);
                    const float wyz = __fmul_rn(wy, wz);
                    const float w = __fmul_rn(wx, wyz);
                    if (MODE == POI_SYSTEM) {
                        const float *nr = attr + 3 * (size_t)__float_as_int(r.w);
                        const float gx = dx ? wyz : -wyz;
                        const float gy = __fmul_rn(dy ? wx : -wx, wz);
                        const float gz = __fmul_rn(dz ? wx : -wx, wy);
                        float d = __fmul_rn(nr[0], gx);
                        d = __fadd_rn(d, __fmul_rn(nr[1], gy));
                        d = __fadd_rn(d, __fmul_rn(nr[2], gz));
                        acc0 = __fadd_rn(acc0, d);
                        acc1 = __fadd_rn(acc1, w);
                    } else if (MODE == POI_WEIGHT) {
                        acc0 = __fadd_rn(acc0, w);
                    } else {
                        acc0 = __fadd_rn(acc0, __fmul_rn(w, attr[3 * (size_t)__float_as_int(r.w) + channel]));
                    }
                }
            }
        }
    }
    if (MODE == POI_SYSTEM) {
        out0[node] = -__fmul_rn(area, acc0);
        out1[node] = __fmul_rn(__fmul_rn(alpha, area), acc1);
    } else {
        out0[node] = acc0;
    }
}

// sum_{j in N6(i)} (u_i - u_j) over the neighbours inside the grid, and their count
__device__ __forceinline__ float neighbour_diff(const float *__restrict__ u, int N, int i, int j, int k, size_t at, float ui,
                                                int *cnt)
{
    const size_t NN = (size_t)N * N;
    float s = 0.0f;
    int c = 0;
    if (i > 0) s += ui - u[at - NN], c++;
    if (i < N - 1) s += ui - u[at + NN], c++;
    if (j > 0) s += ui - u[at - N], c++;
    if (j < N - 1) s += ui - u[at + N], c++;
    if (k > 0) s += ui - u[at - 1], c++;
    if (k < N - 1) s += ui - u[at + 1], c++;
    *cnt = c;
    return s;
}

// b_i - (coeff * sum (u_i - u_j) + q_i u_i); u == nullptr reads zeros
__device__ __forceinline__ float residual_at(const float *__restrict__ u, const float *__restrict__ b,
                                             const float *__restrict__ q, int N, float coeff, int i, int j, int k)
{
    const size_t at = ((size_t)i * N + j) * N + k;
    if (!u) return b[at];
    const float ui = u[at];
    int c;
    const float d = neighbour_diff(u, N, i, j, k, at, ui, &c);
    return b[at] - fmaf(coeff, d, q[at] * ui);
}

// one colour of red-black Gauss-Seidel: nodes with (i + j + k) % 2 == colour
__global__ void __launch_bounds__(256) poi_smooth_kernel(int N, float coeff, int colour, float *__restrict__ u,
                                                         const float *__restrict__ b, const float *__restrict__ q)
{
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    const int half = N / 2;
    if (t >= (size_t)N * N * half) return;
    const int i = (int)(t / ((size_t)N * half)), j = (int)(t / half % N);
    const int k = 2 * (int)(t % half) + ((i + j + colour) & 1);
    const size_t NN = (size_t)N * N, at = ((size_t)i * N + j) * N + k;
    float s = 0.0f;
    int c = 0;
    if (i > 0) s += u[at - NN], c++;
    if (i < N - 1) s += u[at + NN], c++;
    if (j > 0) s += u[at - N], c++;
    if (j < N - 1) s += u[at + N], c++;
    if (k > 0) s += u[at - 1], c++;
    if (k < N - 1) s += u[at + 1], c++;
    u[at] = fmaf(coeff, s, b[at]) / fmaf(coeff, (float)c, q[at]);
}

// coarse[I] = sum over the 8 children of the fine residual (u == nullptr: of `b` itself); coarse u = 0
__global__ void __launch_bounds__(256) poi_restrict_kernel(int Nc, float coeff, const float *__restrict__ u,
                                                           const float *__restrict__ b, const float *__restrict__ q,
                                                           float *__restrict__ bc, float *__restrict__ uc)
{
    const size_t I = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (I >= (size_t)Nc * Nc * Nc) return;
    const int ci = (int)(I / ((size_t)Nc * Nc)), cj = (int)(I / Nc % Nc), ck = (int)(I % Nc);
    const int N = 2 * Nc;
    float s = 0.0f;
    for (int a = 0; a < 2; a++)
        for (int c = 0; c < 2; c++)
            for (int d = 0; d < 2; d++) s += residual_at(u, b, q, N, coeff, 2 * ci + a, 2 * cj + c, 2 * ck + d);
    bc[I] = s;
    if (uc) uc[I] = 0.0f;
}

// u_fine += cell-centred trilinear interpolation of the coarse correction
__global__ void __launch_bounds__(256) poi_prolong_kernel(int N, float *__restrict__ u, const float *__restrict__ uc)
{
    const size_t at = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (at >= (size_t)N * N * N) return;
    const int Nc = N / 2;
    const int f[3] = {(int)(at / ((size_t)N * N)), (int)(at / N % N), (int)(at % N)};
    int c0[3], c1[3];
    float w0[3];
    for (int a = 0; a < 3; a++) {
        c0[a] = f[a] >> 1;
        const int o = (f[a] & 1) ? c0[a] + 1 : c0[a] - 1;  // the other coarse node nearest this fine node
        c1[a] = min(max(o, 0), Nc - 1);
        w0[a] = 0.75f;
    }
    float s = 0.0f;
    for (int a = 0; a < 2; a++)
        for (int c = 0; c < 2; c++)
            for (int d = 0; d < 2; d++) {
                const float w = (a ? 0.25f : w0[0]) * (c ? 0.25f : w0[1]) * (d ? 0.25f : w0[2]);
                const int x = a ? c1[0] : c0[0], y = c ? c1[1] : c0[1], z = d ? c1[2] : c0[2];
                s = fmaf(w, uc[((size_t)x * Nc + y) * Nc + z], s);
            }
    u[at] += s;
}

// the 4^3 level: one CTA of 64 threads, POI_COARSEST_SWEEPS red-black sweeps in shared memory
__global__ void __launch_bounds__(64) poi_coarsest_kernel(float coeff, float *__restrict__ u, const float *__restrict__ b,
                                                          const float *__restrict__ q)
{
    constexpr int N = 4;
    __shared__ float su[64];
    const int t = threadIdx.x;
    const int i = t >> 4, j = (t >> 2) & 3, k = t & 3;
    su[t] = u[t];
    const float bt = b[t], qt = q[t];
    __syncthreads();
    for (int sweep = 0; sweep < 2 * POI_COARSEST_SWEEPS; sweep++) {
        if (((i + j + k) & 1) == (sweep & 1)) {
            float s = 0.0f;
            int c = 0;
            if (i > 0) s += su[t - 16], c++;
            if (i < N - 1) s += su[t + 16], c++;
            if (j > 0) s += su[t - 4], c++;
            if (j < N - 1) s += su[t + 4], c++;
            if (k > 0) s += su[t - 1], c++;
            if (k < N - 1) s += su[t + 1], c++;
            su[t] = fmaf(coeff, s, bt) / fmaf(coeff, (float)c, qt);
        }
        __syncthreads();
    }
    u[t] = su[t];
}

// Fixed-order sums: thread (block, tid) takes items block * 256 + tid + m * POI_RED_BLOCKS * 256, cta_tree_sum per
// block, then one CTA sums the POI_RED_BLOCKS partials by the same tree.
__global__ void __launch_bounds__(256) poi_residual_sq_kernel(int N, float coeff, const float *__restrict__ u,
                                                              const float *__restrict__ b, const float *__restrict__ q,
                                                              double *__restrict__ partial)
{
    __shared__ double sh[256];
    const size_t total = (size_t)N * N * N, stride = (size_t)POI_RED_BLOCKS * 256;
    double acc = 0.0;
    for (size_t at = (size_t)blockIdx.x * 256 + threadIdx.x; at < total; at += stride) {
        const float r = residual_at(u, b, q, N, coeff, (int)(at / ((size_t)N * N)), (int)(at / N % N), (int)(at % N));
        acc += (double)r * r;
    }
    const double s = cta_tree_sum<256>(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(POI_RED_BLOCKS) poi_final_sum_kernel(double *__restrict__ partial)
{
    __shared__ double sh[POI_RED_BLOCKS];
    const double s = cta_sum_partials<POI_RED_BLOCKS>(POI_RED_BLOCKS, partial, 1, sh);
    if (threadIdx.x == 0) partial[0] = s;
}

// trilinear interpolation of grid [N,N,N] at g = p * scale + offset (clamped to the grid), per point
__global__ void __launch_bounds__(256) poi_interpolate_kernel(int N, const float *__restrict__ grid, int64_t m,
                                                              const float *__restrict__ pts, int stride, float scale,
                                                              float offset, float *__restrict__ values,
                                                              double *__restrict__ partial)
{
    __shared__ double sh[256];
    const int64_t step = (int64_t)POI_RED_BLOCKS * 256;
    double acc = 0.0;
    for (int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x; s < m; s += step) {
        int l[3];
        float t[3];
        for (int a = 0; a < 3; a++) {
            const float g = fmaf(pts[s * stride + a], scale, offset);
            l[a] = lower_node(g, N);
            t[a] = fminf(fmaxf(g - (float)l[a], 0.0f), 1.0f);
        }
        float v = 0.0f;
        for (int a = 0; a < 2; a++)
            for (int c = 0; c < 2; c++)
                for (int d = 0; d < 2; d++) {
                    const float w = (a ? t[0] : 1.0f - t[0]) * (c ? t[1] : 1.0f - t[1]) * (d ? t[2] : 1.0f - t[2]);
                    v = fmaf(w, grid[((size_t)(l[0] + a) * N + l[1] + c) * N + l[2] + d], v);
                }
        if (values) values[s] = v;
        acc += v;
    }
    if (partial) {
        const double total = cta_tree_sum<256>(acc, sh);
        if (threadIdx.x == 0) partial[blockIdx.x] = total;
    }
}

static bool poi_side_ok(int32_t N) { return N >= 4 && N <= 1024 && (N & (N - 1)) == 0; }

static int read_sum(double *partial, double *out, cudaStream_t st)
{
    SGR_LAUNCH(K_MISC, st, poi_final_sum_kernel<<<1, POI_RED_BLOCKS, 0, st>>>(partial));
    SGR_CUDA(cudaMemcpyAsync(out, partial, sizeof(double), cudaMemcpyDeviceToHost, st));
    SGR_CUDA(cudaStreamSynchronize(st));
    return SGR_OK;
}

static int residual_norm(int N, float coeff, const float *u, const float *b, const float *q, double *partial,
                         double *norm, cudaStream_t st)
{
    SGR_LAUNCH(K_MISC, st, poi_residual_sq_kernel<<<POI_RED_BLOCKS, 256, 0, st>>>(N, coeff, u, b, q, partial));
    double sq = 0.0;
    const int rc = read_sum(partial, &sq, st);
    if (rc) return rc;
    *norm = sqrt(sq);
    return SGR_OK;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_poisson_bin(int32_t n, const float *points, int32_t N, float ox, float oy, float oz, float inv_h,
                    uint32_t *starts, float *binned, uint32_t *keys, float *records, uint32_t *hist,
                    uint32_t *block_sums, int64_t *n_occupied, void *stream)
{
    if (n <= 0 || !poi_side_ok(N) || !(inv_h > 0.0f)) {
        set_error("sgr_poisson_bin: need n > 0, N a power of two in [4, 1024] and inv_h > 0 (n=%d N=%d)", n, N);
        return SGR_EINVAL;
    }
    if (!points || !starts || !binned || !keys || !records || !hist || !block_sums || !n_occupied ||
        !aligned16(binned) || !aligned16(records)) {
        set_error("sgr_poisson_bin: null or misaligned pointer (binned and records need 16 bytes)");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const size_t nbins = (size_t)N * N * N;
    const int ntiles = (n + POI_RADIX_TILE - 1) / POI_RADIX_TILE;
    int bits = 0;
    while (((size_t)1 << bits) < nbins) bits++;
    const int passes = (bits + 7) / 8;
    // the passes alternate between the two buffers and end in `binned`
    float4 *rec[2] = {(float4 *)(passes & 1 ? records : binned), (float4 *)(passes & 1 ? binned : records)};
    uint32_t *key[2] = {keys, keys + n};
    SGR_CUDA(cudaMemsetAsync(starts, 0, nbins * 4, st));
    SGR_LAUNCH(K_MISC, st, poi_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(n, points, ox, oy, oz, inv_h, N, key[0],
                                                                                rec[0], starts));
    exclusive_scan(K_MISC, nbins, starts, starts, block_sums, starts, st);
    for (int p = 0; p < passes; p++) {
        const int a = p & 1;
        SGR_LAUNCH(K_MISC, st, poi_radix_hist_kernel<<<ntiles, POI_RADIX_TILE, 0, st>>>(n, key[a], 8 * p, ntiles, hist));
        exclusive_scan(K_MISC, 256 * ntiles, hist, hist, block_sums, hist, st);
        SGR_LAUNCH(K_MISC, st, poi_radix_scatter_kernel<<<ntiles, POI_RADIX_TILE, 0, st>>>(
                                   n, key[a], rec[a], 8 * p, ntiles, hist, key[a ^ 1], rec[a ^ 1]));
    }
    SGR_CUDA(cudaMemsetAsync(block_sums, 0, 4, st));
    SGR_LAUNCH(K_MISC, st, poi_occupied_kernel<<<blocks_for(n, 256), 256, 0, st>>>(n, key[passes & 1], block_sums));
    uint32_t occ = 0;
    SGR_CUDA(cudaMemcpyAsync(&occ, block_sums, 4, cudaMemcpyDeviceToHost, st));
    SGR_CUDA(cudaStreamSynchronize(st));
    *n_occupied = occ;
    return SGR_OK;
}

int sgr_poisson_splat(int32_t N, int32_t n, const uint32_t *starts, const float *binned, int32_t mode, const float *attr,
                      int32_t channel, float area, float alpha, float *out0, float *out1, void *stream)
{
    if (!poi_side_ok(N) || n <= 0 || mode < POI_SYSTEM || mode > POI_ATTRIBUTE || channel < 0 || channel > 2) {
        set_error("sgr_poisson_splat: need N a power of two in [4, 1024], n > 0, mode 0-2 and channel 0-2 "
                  "(N=%d n=%d mode=%d channel=%d)", N, n, mode, channel);
        return SGR_EINVAL;
    }
    if (!starts || !binned || !out0 || (mode != POI_WEIGHT && !attr) || (mode == POI_SYSTEM && !out1) ||
        !aligned16(binned)) {
        set_error("sgr_poisson_splat: null or misaligned pointer (binned needs 16 bytes)");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned g = blocks_for((size_t)N * N * N, 256);
    const float4 *bn = (const float4 *)binned;
    const uint32_t un = (uint32_t)n;
    if (mode == POI_SYSTEM)
        SGR_LAUNCH(K_MISC, st, poi_splat_kernel<POI_SYSTEM><<<g, 256, 0, st>>>(N, un, starts, bn, attr, 0, area, alpha, out0,
                                                                              out1));
    else if (mode == POI_WEIGHT)
        SGR_LAUNCH(K_MISC, st, poi_splat_kernel<POI_WEIGHT><<<g, 256, 0, st>>>(N, un, starts, bn, nullptr, 0, 0.f, 0.f, out0,
                                                                              nullptr));
    else
        SGR_LAUNCH(K_MISC, st, poi_splat_kernel<POI_ATTRIBUTE><<<g, 256, 0, st>>>(N, un, starts, bn, attr, channel, 0.f, 0.f,
                                                                                 out0, nullptr));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_poisson_coarsen(int32_t N, const float *fine, float *coarse, void *stream)
{
    if (!poi_side_ok(N) || N < 8 || !fine || !coarse) {
        set_error("sgr_poisson_coarsen: need N a power of two in [8, 1024] and non-null pointers (N=%d)", N);
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int Nc = N / 2;
    SGR_LAUNCH(K_MISC, st, poi_restrict_kernel<<<blocks_for((size_t)Nc * Nc * Nc, 256), 256, 0, st>>>(
                               Nc, 1.0f, nullptr, fine, nullptr, coarse, nullptr));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_poisson_residual_norm(int32_t N, float coeff, const float *u, const float *b, const float *q, double *partial,
                              double *norm, void *stream)
{
    if (!poi_side_ok(N) || !(coeff > 0.0f) || !b || (u && !q) || !partial || !norm) {
        set_error("sgr_poisson_residual_norm: need N a power of two in [4, 1024], coeff > 0 and non-null b, partial, "
                  "norm (q too when u is given) (N=%d)", N);
        return SGR_EINVAL;
    }
    return residual_norm(N, coeff, u, b, q, partial, norm, (cudaStream_t)stream);
}

int sgr_poisson_vcycle(int32_t depth, float *const *u, float *const *b, const float *const *q, double *partial,
                       double *norm, void *stream)
{
    if (depth < 3 || depth > 10 || !u || !b || !q || !partial || !norm) {
        set_error("sgr_poisson_vcycle: need 3 <= depth <= 10 and non-null level arrays, partial and norm (depth=%d)",
                  depth);
        return SGR_EINVAL;
    }
    const int L = depth - 1;  // levels 2^depth .. 4
    for (int l = 0; l < L; l++)
        if (!u[l] || !b[l] || !q[l]) {
            set_error("sgr_poisson_vcycle: null grid at level %d", l);
            return SGR_EINVAL;
        }
    cudaStream_t st = (cudaStream_t)stream;
    auto smooth = [&](int l, int sweeps) {
        const int N = (1 << depth) >> l;
        const unsigned g = blocks_for((size_t)N * N * N / 2, 256);
        for (int s = 0; s < sweeps; s++)
            for (int c = 0; c < 2; c++)
                SGR_LAUNCH(K_MISC, st, poi_smooth_kernel<<<g, 256, 0, st>>>(N, (float)(1 << l), c, u[l], b[l], q[l]));
    };
    for (int l = 0; l < L - 1; l++) {
        const int N = (1 << depth) >> l, Nc = N / 2;
        smooth(l, 2);
        SGR_LAUNCH(K_MISC, st, poi_restrict_kernel<<<blocks_for((size_t)Nc * Nc * Nc, 256), 256, 0, st>>>(
                                   Nc, (float)(1 << l), u[l], b[l], q[l], b[l + 1], u[l + 1]));
    }
    SGR_LAUNCH(K_MISC, st, poi_coarsest_kernel<<<1, 64, 0, st>>>((float)(1 << (L - 1)), u[L - 1], b[L - 1], q[L - 1]));
    for (int l = L - 2; l >= 0; l--) {
        const int N = (1 << depth) >> l;
        SGR_LAUNCH(K_MISC, st, poi_prolong_kernel<<<blocks_for((size_t)N * N * N, 256), 256, 0, st>>>(N, u[l], u[l + 1]));
        smooth(l, 2);
    }
    SGR_CUDA(cudaGetLastError());
    return residual_norm(1 << depth, 1.0f, u[0], b[0], q[0], partial, norm, st);
}

int sgr_poisson_interpolate(int32_t N, const float *grid, int64_t m, const float *points, int32_t stride, float scale,
                            float offset, float *values, double *partial, double *sum, void *stream)
{
    if (!poi_side_ok(N) || m < 0 || stride < 3 || (sum && !partial)) {
        set_error("sgr_poisson_interpolate: need N a power of two in [4, 1024], m >= 0, stride >= 3, and partial "
                  "with sum (N=%d m=%lld stride=%d)", N, (long long)m, stride);
        return SGR_EINVAL;
    }
    if (!grid || (m > 0 && !points) || (!values && !sum)) {
        set_error("sgr_poisson_interpolate: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (m > 0)
        SGR_LAUNCH(K_MISC, st, poi_interpolate_kernel<<<POI_RED_BLOCKS, 256, 0, st>>>(
                                   N, grid, m, points, stride, scale, offset, values, sum ? partial : nullptr));
    else if (sum)
        SGR_CUDA(cudaMemsetAsync(partial, 0, POI_RED_BLOCKS * sizeof(double), st));
    SGR_CUDA(cudaGetLastError());
    return sum ? read_sum(partial, sum, st) : SGR_OK;
}

}  // extern "C"
