// sgr_scan.cu -- device-wide exclusive scan of uint32 counts (cell, bin, vertex and piece offsets).
//
// Three kernels: each 1024-thread block sums 4096 counts (4 per thread) into block_sums, one CTA scans the block sums in
// chunks of 1024, and each block scans its counts again from its offset.  The counts are read twice and the offsets
// written once.
#include "sgr_reduce.cuh"
#include "sgr_scan.cuh"

namespace sgr {

// A thread's four counts and the CTA's exclusive scan of their sums (cta_exclusive_scan)
template <typename T>
__device__ __forceinline__ T scan_load4(size_t n, size_t i0, const uint32_t *counts, T v[4], T *s_w)
{
    T sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        v[k] = (i0 + k < n) ? counts[i0 + k] : 0u;
        sum += v[k];
    }
    return cta_exclusive_scan(sum, s_w);
}

template <typename T>
__global__ void __launch_bounds__(1024) scan_reduce_kernel(size_t n, const uint32_t *__restrict__ counts,
                                                           T *__restrict__ block_sums)
{
    __shared__ T s_w[32];
    T v[4];
    const T ex = scan_load4(n, ((size_t)blockIdx.x * 1024 + threadIdx.x) * 4, counts, v, s_w);
    if (threadIdx.x == 1023) block_sums[blockIdx.x] = ex + v[0] + v[1] + v[2] + v[3];
}

template <typename T>
__global__ void __launch_bounds__(1024) scan_sums_kernel(int nblocks, T *block_sums)
{
    // single CTA, serial over chunks of 1024 (nblocks <= 4096 for 2^24 counts)
    __shared__ T s_w[32];
    __shared__ T s_carry;
    const int tid = threadIdx.x;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        const T v = (base + tid < nblocks) ? block_sums[base + tid] : 0u;
        const T ex = s_carry + cta_exclusive_scan(v, s_w);
        if (base + tid < nblocks) block_sums[base + tid] = ex;
        __syncthreads();
        if (tid == 1023) s_carry = ex + v;
        __syncthreads();
    }
}

// counts, starts and cursor may alias (in place): a thread loads its four counts before the barriers of
// cta_exclusive_scan and stores only its own four offsets after them
template <typename T>
__global__ void __launch_bounds__(1024) scan_apply_kernel(size_t n, const uint32_t *counts, const T *__restrict__ block_offs,
                                                          T *starts, T *cursor)
{
    __shared__ T s_w[32];
    T v[4];
    const size_t i0 = ((size_t)blockIdx.x * 1024 + threadIdx.x) * 4;
    T run = block_offs[blockIdx.x] + scan_load4(n, i0, counts, v, s_w);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (i0 + k < n) {
            starts[i0 + k] = run;
            if (cursor != starts) cursor[i0 + k] = run;
        }
        run += v[k];
    }
}

template <typename T>
void exclusive_scan(int kind, size_t n, const uint32_t *counts, T *starts, T *block_sums, T *cursor, cudaStream_t st)
{
    const int nblocks = (int)((n + 4095) / 4096);
    SGR_LAUNCH(kind, st, scan_reduce_kernel<T><<<(unsigned)nblocks, 1024, 0, st>>>(n, counts, block_sums));
    SGR_LAUNCH(kind, st, scan_sums_kernel<T><<<1, 1024, 0, st>>>(nblocks, block_sums));
    SGR_LAUNCH(kind, st, scan_apply_kernel<T><<<(unsigned)nblocks, 1024, 0, st>>>(n, counts, block_sums, starts, cursor));
}

template void exclusive_scan<uint32_t>(int, size_t, const uint32_t *, uint32_t *, uint32_t *, uint32_t *, cudaStream_t);
template void exclusive_scan<unsigned long long>(int, size_t, const uint32_t *, unsigned long long *, unsigned long long *,
                                                 unsigned long long *, cudaStream_t);

}  // namespace sgr
