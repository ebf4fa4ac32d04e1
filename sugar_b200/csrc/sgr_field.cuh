// sgr_field.cuh -- the field's packed Gaussian records and per-neighbour density term, shared by sgr_field.cu and the
// density grid of sgr_mcubes.cu (so that both give the same bits for the same neighbour); and the pieces of the
// neighbour-group kernels of sgr_field.cu and sgr_normal.cu: the smallest-axis normal, its quaternion backward, the
// lane-group sum and the launch by group width.
#pragma once
#include <type_traits>

#include "sgr_internal.cuh"

namespace sgr {

// packed per-Gaussian record, 12 floats:  mu.xyz sig | q.rijk | inv_s.xyz s_min; `kind` profiles the launch
void field_pack(int kind, int P, const float *points, const float *scaling, const float *quats, const float *strengths,
                float4 *rec, cudaStream_t st);

#ifdef __CUDACC__
struct Rot {
    float m[3][3];  // row-major R[row][col]
    float ts;       // two_s = 2 / |q|^2
};
__device__ __forceinline__ Rot quat_to_rot(float4 q)
{
    const float r = q.x, i = q.y, j = q.z, k = q.w;
    Rot o;
    o.ts = 2.0f / (r * r + i * i + j * j + k * k);
    const float ts = o.ts;
    o.m[0][0] = 1 - ts * (j * j + k * k);
    o.m[0][1] = ts * (i * j - k * r);
    o.m[0][2] = ts * (i * k + j * r);
    o.m[1][0] = ts * (i * j + k * r);
    o.m[1][1] = 1 - ts * (i * i + k * k);
    o.m[1][2] = ts * (j * k - i * r);
    o.m[2][0] = ts * (i * k - j * r);
    o.m[2][1] = ts * (j * k + i * r);
    o.m[2][2] = 1 - ts * (i * i + j * j);
    return o;
}

// density_factor * strength * exp(-1/2 |L^-T (x - mu)|^2), the squared norm clamped to [0, 1e8]
// (sugar_model.py:1359-1362), from the Gaussian's three packed records
__device__ __forceinline__ float field_term(float x0, float x1, float x2, float4 r0, float4 r1, float4 r2,
                                            float density_factor)
{
    const Rot R = quat_to_rot(r1);
    const float sh0 = x0 - r0.x, sh1 = x1 - r0.y, sh2 = x2 - r0.z;
    const float w0 = (R.m[0][0] * sh0 + R.m[1][0] * sh1 + R.m[2][0] * sh2) * r2.x;
    const float w1 = (R.m[0][1] * sh0 + R.m[1][1] * sh1 + R.m[2][1] * sh2) * r2.y;
    const float w2 = (R.m[0][2] * sh0 + R.m[1][2] * sh1 + R.m[2][2] * sh2) * r2.z;
    const float d2 = fminf(fmaxf(w0 * w0 + w1 * w1 + w2 * w2, 0.f), 1e8f);
    return density_factor * r0.w * expf(-0.5f * d2);
}

// dL/dq from A = dL/dR, R = I + ts * E(q) with ts = two_s = 2 / |q|^2 (pytorch3d's quaternion_to_matrix)
__device__ __forceinline__ float4 rot_backward(const float (&A)[3][3], float4 q, float ts)
{
    const float qr = q.x, qi = q.y, qj = q.z, qk = q.w;
    const float dts = A[0][0] * -(qj * qj + qk * qk) + A[0][1] * (qi * qj - qk * qr) + A[0][2] * (qi * qk + qj * qr) +
                      A[1][0] * (qi * qj + qk * qr) + A[1][1] * -(qi * qi + qk * qk) + A[1][2] * (qj * qk - qi * qr) +
                      A[2][0] * (qi * qk - qj * qr) + A[2][1] * (qj * qk + qi * qr) + A[2][2] * -(qi * qi + qj * qj);
    const float c = -ts * ts * dts;  // d ts / d q_c = -ts^2 q_c
    const float dqr = ts * (-qk * A[0][1] + qj * A[0][2] + qk * A[1][0] - qi * A[1][2] - qj * A[2][0] + qi * A[2][1]) + c * qr;
    const float dqi = ts * (qj * (A[0][1] + A[1][0]) + qk * (A[0][2] + A[2][0]) + qr * (A[2][1] - A[1][2]) -
                            2.f * qi * (A[1][1] + A[2][2])) + c * qi;
    const float dqj = ts * (qi * (A[0][1] + A[1][0]) + qr * (A[0][2] - A[2][0]) + qk * (A[1][2] + A[2][1]) -
                            2.f * qj * (A[0][0] + A[2][2])) + c * qj;
    const float dqk = ts * (qr * (A[1][0] - A[0][1]) + qi * (A[0][2] + A[2][0]) + qj * (A[1][2] + A[2][1]) -
                            2.f * qk * (A[0][0] + A[1][1])) + c * qk;
    return make_float4(dqr, dqi, dqj, dqk);
}

// index of the first minimum of a scaling row, the tie rule of torch.min(dim)
__device__ __forceinline__ int smallest_index(float s0, float s1, float s2)
{
    int a = 0;
    float smin = s0;
    if (s1 < smin) smin = s1, a = 1;
    if (s2 < smin) a = 2;
    return a;
}

// A Gaussian's normal as SuGaR's get_normals / get_smallest_axis take it: column `col` of R(q), `col` the first
// minimum of its scaling row `s`.  The index comes from the float scaling, not a clamped 1/s, so no clamp can change
// the pick.
struct SmallestAxis {
    int col;
    float n[3];
    float ts;  // two_s of q
};

__device__ __forceinline__ SmallestAxis smallest_axis(const float *s, float4 q)
{
    SmallestAxis a;
    a.col = smallest_index(s[0], s[1], s[2]);
    const Rot R = quat_to_rot(q);
    a.ts = R.ts;
#pragma unroll
    for (int i = 0; i < 3; i++) a.n[i] = a.col == 0 ? R.m[i][0] : (a.col == 1 ? R.m[i][1] : R.m[i][2]);
    return a;
}

// dL/dq from dL/dn of that normal: dL/dR is dn in column `col` and zero elsewhere
__device__ __forceinline__ float4 smallest_axis_backward(const SmallestAxis &a, float4 q, const float (&dn)[3])
{
    float A[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        A[i][0] = a.col == 0 ? dn[i] : 0.f;
        A[i][1] = a.col == 1 ? dn[i] : 0.f;
        A[i][2] = a.col == 2 ? dn[i] : 0.f;
    }
    return rot_backward(A, q, a.ts);
}

// The neighbour-group kernels give K neighbours to a group of G = group_width(K) lanes: lane l sums terms l, l + G, ...
// in order, then the lanes are reduced by group_sum's xor butterfly (lane 0 gets s[0] + s[G/2] first, and so on down).
__host__ __device__ __forceinline__ int group_width(int K)
{
    int G = 1;
    while (G < K && G < 32) G <<= 1;
    return G;
}

template <int G>
__device__ __forceinline__ float group_sum(float v)
{
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// f(std::integral_constant<int, G>{}) for G = group_width(K): one launch site per kernel template
template <class F>
void with_group_width(int K, F f)
{
    switch (group_width(K)) {
        case 1: f(std::integral_constant<int, 1>{}); break;
        case 2: f(std::integral_constant<int, 2>{}); break;
        case 4: f(std::integral_constant<int, 4>{}); break;
        case 8: f(std::integral_constant<int, 8>{}); break;
        case 16: f(std::integral_constant<int, 16>{}); break;
        default: f(std::integral_constant<int, 32>{}); break;
    }
}
#endif

}  // namespace sgr
