// sgr_compose.cu -- SH colours at a per-group rotated view direction, for the compositor (sugar_b200/compose.py).
//
// SuGaRCompositor.render_image_gaussian_rasterizer (sugar_compositor.py:139-151) turns the view direction of a rigidly
// moved model into the model's own frame, normalize(p - campos) @ sh_rotation, before eval_sh, so that its
// view-dependent colour turns with it.  The rasterizer evaluates SH at the unrotated direction only, so these colours
// enter it as colors_precomp.  One thread per Gaussian; the direction, basis, channel sum and clamp are the forward's
// own (sgr_sh.cuh, sgr_forward.cu), so R = I reproduces the in-kernel colour bit for bit.
#include "sgr_sh.cuh"

namespace sgr {

__global__ void __launch_bounds__(256) sh_colors_rotated_kernel(int P, int M, int deg, const float *__restrict__ means,
                                                                const float *__restrict__ shs,
                                                                const float *__restrict__ campos, int G,
                                                                const int64_t *__restrict__ group_start,
                                                                const float *__restrict__ group_rot,
                                                                float *__restrict__ colors)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int g = 0;
    while (g + 1 < G && i >= group_start[g + 1]) g++;  // G is the number of composited models: a handful
    const float *R = group_rot + 9 * g;
    const f3 d = sh_dir(means[3 * (size_t)i], means[3 * (size_t)i + 1], means[3 * (size_t)i + 2], campos[0], campos[1],
                        campos[2]);
    f3 dr;  // the row vector d times R
    dr.x = __fmaf_rn(d.z, R[6], __fmaf_rn(d.y, R[3], __fmul_rn(d.x, R[0])));
    dr.y = __fmaf_rn(d.z, R[7], __fmaf_rn(d.y, R[4], __fmul_rn(d.x, R[1])));
    dr.z = __fmaf_rn(d.z, R[8], __fmaf_rn(d.y, R[5], __fmul_rn(d.x, R[2])));
    const float *row = shs + (size_t)i * M * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float v = sh_channel(deg, dr, [&](int k) { return row[k * 3 + c]; });
        colors[3 * (size_t)i + c] = v < -0.5f ? 0.0f : __fadd_rn(v, 0.5f);  // the forward's clamp (forward.cu:63-70)
    }
}

}  // namespace sgr

using namespace sgr;

extern "C" int sgr_sh_colors_rotated(int32_t P, int32_t M, int32_t sh_degree, const float *means, const float *shs,
                                     const float *campos, int32_t G, const int64_t *group_start, const float *group_rot,
                                     float *colors, void *stream)
{
    if (P < 0 || G <= 0 || sh_degree < 0 || sh_degree > 3 || M < (sh_degree + 1) * (sh_degree + 1) ||
        (P > 0 && (!means || !shs || !campos || !group_start || !group_rot || !colors))) {
        set_error("bad arguments to sgr_sh_colors_rotated");
        return SGR_EINVAL;
    }
    if (P == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               sh_colors_rotated_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, M, sh_degree, means, shs, campos, G,
                                                                         group_start, group_rot, colors));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}
