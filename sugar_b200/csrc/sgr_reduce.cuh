// sgr_reduce.cuh -- the warp, CTA and partial-sum primitives every kernel sums and scans with.
//
// Each helper fixes one summation order, so a kernel that calls it gives the same bits from run to run and the
// float and double results stay reproducible; a caller that needs a different order needs a different helper.
#pragma once

namespace sgr {

// Sum over the warp's 32 lanes by an xor butterfly (16, 8, 4, 2, 1): every lane gets the same value.
template <typename T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Inclusive prefix sum over the warp's lanes (shuffles up by 1, 2, 4, 8, 16): lane i gets v_0 + ... + v_i.
template <typename T>
__device__ __forceinline__ T warp_inclusive_scan(T v)
{
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// Exclusive prefix sum of v over a CTA of 1024 threads: each warp scans its lanes, then warp 0 scans the 32 warp
// totals.  s_w is 32 shared entries; every thread must call, and s_w is free again after the caller's next barrier.
// The CTA total is the last thread's result plus its v.
template <typename T>
__device__ __forceinline__ T cta_exclusive_scan(T v, T *s_w)
{
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const T inc = warp_inclusive_scan(v);
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const T w = s_w[lane];
        s_w[lane] = warp_inclusive_scan(w) - w;
    }
    __syncthreads();
    return s_w[wid] + inc - v;
}

// Sum of v over a CTA of NT threads: warp_sum per warp, then thread 0 adds the NT / 32 warp sums in warp order,
// starting from 0.  red is NT / 32 shared entries; the result is valid in thread 0 only.  The thread index is the
// linear one, so a 2-D block of 32-wide rows has one warp per row.
template <int NT, typename T>
__device__ __forceinline__ T cta_sum_by_warps(T v, T *red)
{
    const int t = threadIdx.y * blockDim.x + threadIdx.x;
    v = warp_sum(v);
    if ((t & 31) == 0) red[t >> 5] = v;
    __syncthreads();
    T s = 0;
    if (t == 0) {
#pragma unroll
        for (int w = 0; w < NT / 32; w++) s += red[w];
    }
    return s;
}

// Sum of v over a CTA of NT threads (a power of two) by a halving tree in sh[NT]: sh[t] += sh[t + w] for w = NT / 2
// down to 1.  Every thread gets the sum.
template <int NT>
__device__ __forceinline__ double cta_tree_sum(double v, double *sh)
{
    const int t = threadIdx.x;
    sh[t] = v;
    __syncthreads();
#pragma unroll
    for (int w = NT / 2; w > 0; w >>= 1) {
        if (t < w) sh[t] += sh[t + w];
        __syncthreads();
    }
    return sh[0];
}

// Sum of the n doubles p[0], p[stride], ... by one CTA of NT threads: thread t adds items t, t + NT, ... to 0.0, then
// cta_tree_sum.  Every thread gets the sum.
template <int NT>
__device__ __forceinline__ double cta_sum_partials(int n, const double *__restrict__ p, int stride, double *sh)
{
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += NT) s += p[(size_t)i * stride];
    return cta_tree_sum<NT>(s, sh);
}

// One CTA of NT threads: out[0] = (float)(sum of partials[0..n) * scale), the sum by cta_sum_partials.  The mesh
// losses' second pass over their per-CTA sums.
template <int NT>
__global__ void __launch_bounds__(NT) sum_partials_kernel(int n, double scale, const double *__restrict__ partials,
                                                          float *__restrict__ out)
{
    __shared__ double sh[NT];
    const double s = cta_sum_partials<NT>(n, partials, 1, sh);
    if (threadIdx.x == 0) out[0] = (float)(s * scale);
}

}  // namespace sgr
