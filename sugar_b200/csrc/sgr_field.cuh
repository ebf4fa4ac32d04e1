// sgr_field.cuh -- the field's packed Gaussian records and per-neighbour density term, shared by sgr_field.cu and the
// density grid of sgr_mcubes.cu (so that both give the same bits for the same neighbour).
#pragma once
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

// The field kernels give K neighbours to a group of G = group_width(K) lanes: lane l sums terms l, l + G, ... in
// order, then the lanes are reduced by an xor butterfly (lane 0 gets s[0] + s[G/2] first, and so on down).
__host__ __device__ __forceinline__ int group_width(int K)
{
    int G = 1;
    while (G < K && G < 32) G <<= 1;
    return G;
}
#endif

}  // namespace sgr
