// sgr_texture.cu -- the refined mesh's UV texture: initial texels from the bound Gaussians and a per-view bake of
// rendered colours over the mesh z-buffer.
//
// Replaces extract_texture_image_and_uv_from_gaussians (sugar_scene/sugar_model.py:2464-2677, square_size s, n_sh 1,
// texture_with_gaussian_renders) without pytorch3d.  The UV layout is plain torch (sugar_b200/texture.py); square k
// = (a, b) = (k / n_sq, k % n_sq) of the T x T map (T = s n_sq) holds face 2k (bottom) and 2k + 1 (top).
//
// texture_init_kernel, one thread per texel of the final [T,T,3] image (every texel written once, coalesced):
//   final (row, col) is pre-transpose (i, j) = (col, T-1-row) (the reference's transpose + flip(0)); (ti, tj) =
//   (i % s, j % s) belongs to the bottom face when tj <= ti < s-1, to the top face when ti < tj, else to none (0.5).
//   The face's texel point is the barycentric combination with the fixed weights of :2563-2576 (they extrapolate past
//   the triangle), its density under each of the face's n Gaussians exp(-1/2 clamp(|diag(1/clamp(s,1e-8)) R^T
//   (x - mu)|^2, 0, 1e8)) and the texel takes SH2RGB(sh_dc) of the argmax Gaussian (torch's argmax: NaN wins, ties
//   go to the first index).  float32 throughout, each operation rounded on its own (no contraction into fma), in the
//   order the reference's torch ops evaluate on the CPU.
//
// Per-view bake, two kernels over the H*W pixels, no float atomics:
//   texture_claim_kernel  pixels with pix_to_face >= 0 and zbuf > 0: the face's perspective-correct barycentrics b'
//                         at the pixel's sample point, in double (the z-buffer's projection: view z, projmatrix /
//                         (w + 1e-7), ndc2pix), then the UV in float32 as pytorch3d's interpolate_face_attributes
//                         (fma chain from 0 over the three corners), then TexturesUV's nearest lookup -- grid_sample
//                         with align_corners, border padding, the map flipped in y: g = 2u - 1, ix = ((g + 1) / 2)
//                         (T-1), clamped to [0, T-1], rounded half to even; col = ix(u), row = T-1 - ix(v).  Stores
//                         the texel in pix_texel and atomicMax'es the pixel index into owner[texel] (preset to -1).
//   texture_add_kernel    the pixel that owns its texel adds its clamped RGB to sum[texel] and 1 to count[texel],
//                         and resets owner[texel] to -1 for the next view.
// A texel has one writer per view and views are added in call order, so the float32 sums are the reference's
// ((0 + c_1) + c_2) + ... whenever each view's pixel on a texel is the same; of several pixels of one view on one
// texel the highest row-major index is kept (the reference's non-accumulating index_put keeps an unspecified one).
#include <math.h>

#include "sgr_internal.cuh"

namespace sgr {

constexpr int TEX_THREADS = 256;
constexpr float SH_C0 = 0.28209479177387814f;

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }

__global__ void __launch_bounds__(TEX_THREADS) texture_init_kernel(int F, int n, int V, int s, int n_sq, int T,
                                                                   const float *__restrict__ verts,
                                                                   const long long *__restrict__ faces,
                                                                   const float *__restrict__ points,
                                                                   const float *__restrict__ scaling,
                                                                   const float4 *__restrict__ quats,
                                                                   const float *__restrict__ sh_dc,
                                                                   float *__restrict__ tex)
{
    const long long idx = (long long)blockIdx.x * TEX_THREADS + threadIdx.x;
    if (idx >= (long long)T * T) return;
    const int row = (int)(idx / T), col = (int)(idx % T);
    const int i = col, j = T - 1 - row;
    const int ti = i % s, tj = j % s;
    const long long k = (long long)(i / s) * n_sq + j / s;
    const bool bottom = tj <= ti && ti < s - 1, top = ti < tj;
    const long long f = 2 * k + (top ? 1 : 0);
    float out[3] = {0.0f, 0.0f, 0.0f};   // SH2RGB(0) = 0.5 where no face owns the texel
    if ((bottom || top) && f < F) {
        // weights (:2563-2576): bottom ((s-2-ti), (tj-1)) / (s-3), top ((ti-1), (s-1-tj)) / (s-3), b0 = 1 - (b1 + b2)
        const float den = (float)(s - 3);
        const float b1 = __fdiv_rn(bottom ? (float)(s - 2 - ti) : (float)(ti - 1), den);
        const float b2 = __fdiv_rn(bottom ? (float)(tj - 1) : (float)(s - 1 - tj), den);
        const float bw[3] = {fsub(1.0f, fadd(b1, b2)), b1, b2};
        float x[3] = {0.0f, 0.0f, 0.0f};
        bool ok = true;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const long long vid = __ldg(faces + 3 * f + c);
            ok = ok && vid >= 0 && vid < V;
            const float *p = verts + 3 * (ok ? vid : 0);
#pragma unroll
            for (int d = 0; d < 3; d++) x[d] = c == 0 ? fmul(bw[0], p[d]) : fadd(x[d], fmul(bw[c], p[d]));
        }
        if (ok) {
            int best_m = 0;
            float best = 0.0f;
            for (int m = 0; m < n; m++) {
                const long long g = f * n + m;
                const float4 q = __ldg(quats + g);
                // pytorch3d quaternion_to_matrix (real part first)
                const float r = q.x, qi = q.y, qj = q.z, qk = q.w;
                const float two_s = __fdiv_rn(2.0f, fadd(fadd(fadd(fmul(r, r), fmul(qi, qi)), fmul(qj, qj)), fmul(qk, qk)));
                float R[3][3];
                R[0][0] = fsub(1.0f, fmul(two_s, fadd(fmul(qj, qj), fmul(qk, qk))));
                R[0][1] = fmul(two_s, fsub(fmul(qi, qj), fmul(qk, r)));
                R[0][2] = fmul(two_s, fadd(fmul(qi, qk), fmul(qj, r)));
                R[1][0] = fmul(two_s, fadd(fmul(qi, qj), fmul(qk, r)));
                R[1][1] = fsub(1.0f, fmul(two_s, fadd(fmul(qi, qi), fmul(qk, qk))));
                R[1][2] = fmul(two_s, fsub(fmul(qj, qk), fmul(qi, r)));
                R[2][0] = fmul(two_s, fsub(fmul(qi, qk), fmul(qj, r)));
                R[2][1] = fmul(two_s, fadd(fmul(qj, qk), fmul(qi, r)));
                R[2][2] = fsub(1.0f, fmul(two_s, fadd(fmul(qi, qi), fmul(qj, qj))));
                float sh[3], dist = 0.0f;
#pragma unroll
                for (int d = 0; d < 3; d++) sh[d] = fsub(x[d], points[3 * g + d]);
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    // get_covariance(return_sqrt, inverse_scales): M = R * (1 / clamp(s, 1e-8))[None, :]; (M^T shift)_c
                    const float inv_s = __fdiv_rn(1.0f, fmaxf(scaling[3 * g + c], 1e-8f));
                    const float w = fadd(fadd(fmul(fmul(R[0][c], inv_s), sh[0]), fmul(fmul(R[1][c], inv_s), sh[1])),
                                         fmul(fmul(R[2][c], inv_s), sh[2]));
                    dist = c == 0 ? fmul(w, w) : fadd(dist, fmul(w, w));
                }
                if (!isnan(dist)) dist = fminf(fmaxf(dist, 0.0f), 1e8f);   // torch.clamp keeps NaN
                const float dens = expf(fmul(-0.5f, dist));
                if (m == 0 || (!isnan(best) && (isnan(dens) || dens > best))) {
                    best = dens;
                    best_m = m;
                }
            }
            const float *c = sh_dc + 3 * (f * n + best_m);
            out[0] = c[0];
            out[1] = c[1];
            out[2] = c[2];
        }
    }
    float *o = tex + 3 * idx;
#pragma unroll
    for (int d = 0; d < 3; d++) o[d] = fadd(fmul(out[d], SH_C0), 0.5f);
}

// grid_sample's nearest index along one axis (align_corners, border padding) of the uv coordinate
__device__ __forceinline__ int nearest_index(float uv, int T)
{
    const float g = fsub(fmul(uv, 2.0f), 1.0f);                                   // pixel_uvs * 2.0 - 1.0
    const float ix = fmul(__fdiv_rn(fadd(g, 1.0f), 2.0f), (float)(T - 1));       // grid_sampler_unnormalize
    return (int)rintf(fminf(fmaxf(ix, 0.0f), (float)(T - 1)));                   // clip_coordinates, nearbyint
}

__global__ void __launch_bounds__(TEX_THREADS) texture_claim_kernel(int n_pix, int W, int H, int V, int F, int n_uv, int T,
                                                                    const float *__restrict__ verts,
                                                                    const long long *__restrict__ faces,
                                                                    const float2 *__restrict__ verts_uv,
                                                                    const long long *__restrict__ faces_uv,
                                                                    const float *__restrict__ view,
                                                                    const float *__restrict__ proj,
                                                                    const float *__restrict__ zbuf,
                                                                    const long long *__restrict__ pix_to_face,
                                                                    int *__restrict__ pix_texel, int *__restrict__ owner)
{
    __shared__ float m[32];  // view, proj
    if (threadIdx.x < 16) m[threadIdx.x] = view[threadIdx.x];
    else if (threadIdx.x < 32) m[threadIdx.x] = proj[threadIdx.x - 16];
    __syncthreads();
    const int p = blockIdx.x * TEX_THREADS + threadIdx.x;
    if (p >= n_pix) return;
    int texel = -1;
    const long long f = pix_to_face[p];
    if (f >= 0 && f < F && zbuf[p] > 0.0f) {
        double x[3], y[3], z[3];
        float2 uv[3];
        bool ok = true;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const long long id = __ldg(faces + 3 * f + c), tid = __ldg(faces_uv + 3 * f + c);
            ok = ok && id >= 0 && id < V && tid >= 0 && tid < n_uv;
            const long long vi = ok ? id : 0;
            const double px = verts[3 * vi], py = verts[3 * vi + 1], pz = verts[3 * vi + 2];
            z[c] = px * m[2] + py * m[6] + pz * m[10] + m[14];
            const double hx = px * m[16] + py * m[20] + pz * m[24] + m[28];
            const double hy = px * m[17] + py * m[21] + pz * m[25] + m[29];
            const double hw = px * m[19] + py * m[23] + pz * m[27] + m[31];
            const double inv_w = __drcp_rn(hw + 1e-7);
            x[c] = ((hx * inv_w + 1.0) * W - 1.0) * 0.5;  // ndc2pix
            y[c] = ((hy * inv_w + 1.0) * H - 1.0) * 0.5;
            uv[c] = __ldg(verts_uv + (ok ? tid : 0));
        }
        if (ok) {
            const double sx = p % W, sy = p / W;  // the pixel's sample point in ndc2pix units
            const double area = (x[2] - x[0]) * (y[1] - y[0]) - (y[2] - y[0]) * (x[1] - x[0]);
            double b[3];
#pragma unroll
            for (int e = 0; e < 3; e++) {
                const int a = (e + 1) % 3, c = (e + 2) % 3;
                b[e] = ((sx - x[a]) * (y[c] - y[a]) - (sy - y[a]) * (x[c] - x[a])) / area;
            }
            const double w0 = b[0] * z[1] * z[2], w1 = b[1] * z[0] * z[2], w2 = b[2] * z[0] * z[1];
            const double inv = 1.0 / fmax(w0 + w1 + w2, 1e-8);
            const float bp[3] = {(float)(w0 * inv), (float)(w1 * inv), (float)(w2 * inv)};
            float u = 0.0f, v = 0.0f;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                u = fmaf(bp[c], uv[c].x, u);
                v = fmaf(bp[c], uv[c].y, v);
            }
            texel = (T - 1 - nearest_index(v, T)) * T + nearest_index(u, T);
        }
    }
    pix_texel[p] = texel;
    if (texel >= 0) atomicMax(owner + texel, p);
}

__global__ void __launch_bounds__(TEX_THREADS) texture_add_kernel(int n_pix, const int *__restrict__ pix_texel,
                                                                  const float *__restrict__ image,
                                                                  int *__restrict__ owner, float *__restrict__ sum,
                                                                  int *__restrict__ count)
{
    const int p = blockIdx.x * TEX_THREADS + threadIdx.x;
    if (p >= n_pix) return;
    const int t = pix_texel[p];
    if (t < 0 || owner[t] != p) return;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float v = image[(size_t)c * n_pix + p];
        if (!isnan(v)) v = fminf(fmaxf(v, 0.0f), 1.0f);  // clamp(0, 1) keeps NaN
        sum[3 * (size_t)t + c] = fadd(sum[3 * (size_t)t + c], v);
    }
    count[t] += 1;
    owner[t] = -1;
}

static int tex_blocks(long long n) { return (int)((n + TEX_THREADS - 1) / TEX_THREADS); }

// n_square_per_axis of the layout: int(sqrt(F // 2 + 1) + 1)
static long long squares_per_axis(long long F) { return (long long)(sqrt((double)(F / 2 + 1)) + 1.0); }

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_texture_init(int32_t F, int32_t n, int32_t V, int32_t square_size, int32_t T, const float *verts,
                     const int64_t *faces, const float *points, const float *scaling, const float *quaternions,
                     const float *sh_dc, float *texture, void *stream)
{
    if (F < 0 || n < 1 || V < 0 || square_size < 3 || (long long)F * n > INT32_MAX) {
        set_error("sgr_texture_init: bad sizes F=%d n=%d V=%d square_size=%d (square_size >= 3, F*n <= 2^31 - 1)", F,
                  n, V, square_size);
        return SGR_EINVAL;
    }
    const long long want = (long long)square_size * squares_per_axis(F);
    if (T != want || (long long)T * T > INT32_MAX) {
        set_error("sgr_texture_init: texture size T=%d, the layout of %d faces at square size %d has %lld "
                  "(T*T <= 2^31 - 1)", T, F, square_size, want);
        return SGR_EINVAL;
    }
    if (!texture || (F > 0 && (!verts || !faces || !points || !scaling || !quaternions || !sh_dc))) {
        set_error("sgr_texture_init: null pointer");
        return SGR_EINVAL;
    }
    if ((size_t)quaternions & 15) {
        set_error("sgr_texture_init: quaternions must be 16-byte aligned");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int n_sq = (int)squares_per_axis(F);
    SGR_LAUNCH(K_MISC, st,
               texture_init_kernel<<<tex_blocks((long long)T * T), TEX_THREADS, 0, st>>>(
                   F, n, V, square_size, n_sq, T, verts, (const long long *)faces, points, scaling,
                   (const float4 *)quaternions, sh_dc, texture));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_texture_bake_view(int32_t V, int32_t F, int32_t n_uv, int32_t T, const float *verts, const int64_t *faces,
                          const float *verts_uv, const int64_t *faces_uv, const float *viewmatrix,
                          const float *projmatrix, int32_t W, int32_t H, const float *image, const float *zbuf,
                          const int64_t *pix_to_face, float *tex_sum, int32_t *tex_count, int32_t *owner,
                          int32_t *pix_texel, void *stream)
{
    if (V < 0 || F < 0 || n_uv < 0 || T < 1 || (long long)T * T > INT32_MAX || W < 0 || H < 0 ||
        (long long)W * H > INT32_MAX) {
        set_error("sgr_texture_bake_view: bad sizes V=%d F=%d n_uv=%d T=%d W=%d H=%d (T*T, W*H <= 2^31 - 1)", V, F,
                  n_uv, T, W, H);
        return SGR_EINVAL;
    }
    const long long n_pix = (long long)W * H;
    if (n_pix == 0) return SGR_OK;
    if (!image || !zbuf || !pix_to_face || !tex_sum || !tex_count || !owner || !pix_texel ||
        (F > 0 && (!verts || !faces || !verts_uv || !faces_uv || !viewmatrix || !projmatrix))) {
        set_error("sgr_texture_bake_view: null pointer");
        return SGR_EINVAL;
    }
    if ((size_t)verts_uv & 7) {
        set_error("sgr_texture_bake_view: verts_uv must be 8-byte aligned");
        return SGR_EINVAL;
    }
    if (F == 0) return SGR_OK;  // no face: every pixel is empty
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               texture_claim_kernel<<<tex_blocks(n_pix), TEX_THREADS, 0, st>>>(
                   (int)n_pix, W, H, V, F, n_uv, T, verts, (const long long *)faces, (const float2 *)verts_uv,
                   (const long long *)faces_uv, viewmatrix, projmatrix, zbuf, (const long long *)pix_to_face,
                   pix_texel, owner));
    SGR_LAUNCH(K_MISC, st,
               texture_add_kernel<<<tex_blocks(n_pix), TEX_THREADS, 0, st>>>((int)n_pix, pix_texel, image, owner,
                                                                               tex_sum, tex_count));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
