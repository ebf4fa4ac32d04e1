/*
 * raster_oracle.c -- CPU restatement of the reference Gaussian-splat rasterizer.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (sugar_b200/) may
 * link, import or call this file; only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs use it, as the checker.
 *
 * It restates, function by function, the algorithm of the vendored INRIA
 * diff-gaussian-rasterization inside Anttwo/SuGaR (paths relative to
 * /root/reference/gaussian_splatting/submodules/diff-gaussian-rasterization/):
 *
 *   ref_in_frustum / projection ........ cuda_rasterizer/auxiliary.h:139-164, 58-77
 *   ref_cov3d .......................... cuda_rasterizer/forward.cu:118-152
 *   ref_cov2d .......................... cuda_rasterizer/forward.cu:74-113
 *   ref_sh_color ....................... cuda_rasterizer/forward.cu:20-71
 *   preprocess (per Gaussian) .......... cuda_rasterizer/forward.cu:155-256
 *   ndc2pix / get_rect ................. cuda_rasterizer/auxiliary.h:41-56
 *   scan / duplicate / sort / ranges ... cuda_rasterizer/rasterizer_impl.cu:70-138, 277-317
 *   blend forward ...................... cuda_rasterizer/forward.cu:261-374
 *   blend backward ..................... cuda_rasterizer/backward.cu:399-557
 *   cov2d backward ..................... cuda_rasterizer/backward.cu:144-274
 *   preprocess backward / SH / cov3d ... cuda_rasterizer/backward.cu:20-139, 278-396
 *
 * Floating-point contract.  The tile assignment and the 64-bit sort keys of the
 * reference must be reproduced bit for bit, so every fp32 operation that feeds
 * depth, pixel position, 2-D covariance, radius and tile rectangle is written
 * with explicit fmaf()/plain ops in exactly the fused/unfused pattern that
 * nvcc 12.9 (-fmad=true, the reference's default flags) emits for the reference
 * sources on sm_90a (read off the PTX and SASS of the unmodified sources; the
 * rule is "a*b + c*d + e*f" -> fma(e,f, fma(a,b, c*d)), plus a handful of
 * ptxas-level fusions noted inline).  Compile this file with -ffp-contract=off
 * so that gcc adds no contraction of its own.  expf() here is glibc's; the
 * GPU uses MUFU.EX2, so alpha values can differ in the last ulp: images and
 * gradients are compared with a tolerance, integer/index outputs exactly.
 *
 * Parity pinning: tests/golden/ holds outputs of the UNMODIFIED reference CUDA
 * build (oracle/_ref) run on the GPU, and tests/test_oracle_golden.py checks this
 * file against them.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define TILE 16

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

static inline float fminf_(float a, float b) { return a < b ? a : b; }
static inline float fmaxf_(float a, float b) { return a > b ? a : b; }

/* cvt.rzi.s32.f32: truncate, saturating, NaN -> 0 (CUDA semantics of (int)float). */
static inline int f2i_rz(float f)
{
    if (f != f) return 0;
    if (f >= 2147483648.0f) return INT32_MAX;
    if (f <= -2147483648.0f) return INT32_MIN;
    return (int)f;
}

/* matrix[r] * p.x + matrix[4+r] * p.y + matrix[8+r] * p.z + matrix[12+r]
 * compiled as: fadd( fma(pz, m8, fma(px, m0, py*m4)), m12 )   (auxiliary.h:58-77) */
static inline float xf_row(const float *m, int r, float px, float py, float pz)
{
    float t = py * m[4 + r];
    t = fmaf(px, m[r], t);
    t = fmaf(pz, m[8 + r], t);
    return t + m[12 + r];
}

/* forward.cu:118-152, with mod*scale; glm column-major products, zero terms dropped. */
static void ref_cov3d(const float *scale, float mod, const float *rot, float *cov)
{
    const float sx = mod * scale[0], sy = mod * scale[1], sz = mod * scale[2];
    const float r = rot[0], x = rot[1], y = rot[2], z = rot[3];
    const float yy = y * y, zz = z * z;
    const float rz = r * z, xz = x * z, rx = r * x;
    const float yy_zz = yy + zz;                 /* FADD */
    const float xy_m_rz = fmaf(x, y, -rz);       /* x*y - r*z */
    const float xy_p_rz = fmaf(x, y, rz);        /* x*y + r*z */
    const float ry_p_xz = fmaf(r, y, xz);        /* x*z + r*y */
    const float xz_m_ry = fmaf(-r, y, xz);       /* x*z - r*y */
    const float yz_m_rx = fmaf(y, z, -rx);       /* y*z - r*x */
    const float yz_p_rx = fmaf(y, z, rx);        /* y*z + r*x */
    const float xx_zz = fmaf(x, x, zz);
    const float xx_yy = fmaf(x, x, yy);
    const float R00 = 1.0f - (yy_zz + yy_zz);
    const float R01 = xy_m_rz + xy_m_rz;
    const float R02 = ry_p_xz + ry_p_xz;
    const float R10 = xy_p_rz + xy_p_rz;
    const float R11 = 1.0f - (xx_zz + xx_zz);
    const float R12 = yz_m_rx + yz_m_rx;
    const float R20 = xz_m_ry + xz_m_ry;
    const float R21 = yz_p_rx + yz_p_rx;
    const float R22 = 1.0f - (xx_yy + xx_yy);
    /* M = S * R (glm), nine entries */
    const float a0 = sx * R00, a1 = sy * R01, a2 = sz * R02;
    const float b0 = sx * R10, b1 = sy * R11, b2 = sz * R12;
    const float c0 = sx * R20, c1 = sy * R21, c2 = sz * R22;
    /* Sigma = M^T M; each entry = fma(z-term, fma(x-term, y-term product)) */
    cov[0] = fmaf(a2, a2, fmaf(a0, a0, a1 * a1));
    cov[1] = fmaf(b2, a2, fmaf(b0, a0, b1 * a1));
    cov[2] = fmaf(c2, a2, fmaf(c0, a0, c1 * a1));
    cov[3] = fmaf(b2, b2, fmaf(b0, b0, b1 * b1));
    cov[4] = fmaf(c2, b2, fmaf(c0, b0, c1 * b1));
    cov[5] = fmaf(c2, c2, fmaf(c0, c0, c1 * c1));
}

/* forward.cu:74-113.  Returns cov2D (a,b,c) after the +0.3 low-pass. */
static void ref_cov2d(const float *mean, float focal_x, float focal_y, float tan_fovx, float tan_fovy,
                      const float *c3, const float *vm, float *out)
{
    const float tx0 = xf_row(vm, 0, mean[0], mean[1], mean[2]);
    const float ty0 = xf_row(vm, 1, mean[0], mean[1], mean[2]);
    const float tz = xf_row(vm, 2, mean[0], mean[1], mean[2]);
    const float limx = tan_fovx * 1.3f, limy = tan_fovy * 1.3f;
    const float txtz = tx0 / tz, tytz = ty0 / tz;
    const float cx = fminf_(limx, fmaxf_(-limx, txtz));
    const float cy = fminf_(limy, fmaxf_(-limy, tytz));
    const float tz2 = tz * tz;
    const float J00 = focal_x / tz;
    const float J02 = (focal_x * (cx * (-tz))) / tz2; /* -(focal_x * t.x)/(t.z*t.z), t.x = cx*tz */
    const float J11 = focal_y / tz;
    const float J12 = (focal_y * (cy * (-tz))) / tz2;
    /* T = W * J */
    const float T00 = fmaf(vm[2], J02, vm[0] * J00);
    const float T01 = fmaf(vm[6], J02, vm[4] * J00);
    const float T02 = fmaf(J02, vm[10], vm[8] * J00);
    const float T10 = fmaf(vm[2], J12, J11 * vm[1]);
    const float T11 = fmaf(vm[6], J12, J11 * vm[5]);
    const float T12 = fmaf(J12, vm[10], J11 * vm[9]);
    /* (Vrk^T * T) columns 0 and 1 */
    const float u0 = fmaf(T02, c3[2], fmaf(T00, c3[0], T01 * c3[1]));
    const float v0 = fmaf(T12, c3[2], fmaf(T10, c3[0], T11 * c3[1]));
    const float u1 = fmaf(T02, c3[4], fmaf(T00, c3[1], T01 * c3[3]));
    const float v1 = fmaf(T12, c3[4], fmaf(T10, c3[1], T11 * c3[3]));
    const float u2 = fmaf(T02, c3[5], fmaf(T00, c3[2], T01 * c3[4]));
    const float v2 = fmaf(T12, c3[5], fmaf(T10, c3[2], T11 * c3[4]));
    const float cov00 = fmaf(T02, u2, fmaf(T00, u0, T01 * u1));
    const float cov01 = fmaf(T02, v2, fmaf(T00, v0, T01 * v1));
    const float cov11 = fmaf(T12, v2, fmaf(T10, v0, T11 * v1));
    out[0] = cov00 + 0.3f;
    out[1] = cov01;
    out[2] = cov11 + 0.3f;
}

/* forward.cu:20-71 */
static void ref_sh_color(int deg, int max_coeffs, const float *mean, const float *campos, const float *sh,
                         float *rgb, uint8_t *clamped)
{
    (void)max_coeffs;
    float dx = mean[0] - campos[0], dy = mean[1] - campos[1], dz = mean[2] - campos[2];
    float len = sqrtf(fmaf(dz, dz, fmaf(dx, dx, dy * dy)));
    float x = dx / len, y = dy / len, z = dz / len;
    for (int c = 0; c < 3; c++) {
#define SH(k) sh[(k) * 3 + c]
        float res = SH_C0 * SH(0);
        if (deg > 0) {
            /* ptxas fuses the two subtractions: fma(-(C1*y), sh1, C0*sh0) etc. */
            res = fmaf(-(SH_C1 * y), SH(1), res);
            res = fmaf(SH_C1 * z, SH(2), res);
            res = fmaf(-(SH_C1 * x), SH(3), res);
            if (deg > 1) {
                float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                res = fmaf(SH_C2[0] * xy, SH(4), res);
                res = fmaf(SH_C2[1] * yz, SH(5), res);
                res = fmaf(SH_C2[2] * (((zz + zz) - xx) - yy), SH(6), res);
                res = fmaf(SH_C2[3] * xz, SH(7), res);
                res = fmaf(SH_C2[4] * (xx - yy), SH(8), res);
                if (deg > 2) {
                    const float zz4_xx_yy = fmaf(zz, 4.0f, -xx) - yy;
                    res = fmaf((SH_C3[0] * y) * fmaf(xx, 3.0f, -yy), SH(9), res);
                    res = fmaf((SH_C3[1] * xy) * z, SH(10), res);
                    res = fmaf((SH_C3[2] * y) * zz4_xx_yy, SH(11), res);
                    res = fmaf((SH_C3[3] * z) * fmaf(yy, -3.0f, fmaf(xx, -3.0f, zz + zz)), SH(12), res);
                    res = fmaf((SH_C3[4] * x) * zz4_xx_yy, SH(13), res);
                    res = fmaf((SH_C3[5] * z) * (xx - yy), SH(14), res);
                    res = fmaf((SH_C3[6] * x) * fmaf(yy, -3.0f, xx), SH(15), res);
                }
            }
        }
#undef SH
        res += 0.5f;
        clamped[c] = (res < 0.0f);
        rgb[c] = res < 0.0f ? 0.0f : res;
    }
}

/* auxiliary.h:41-44 (double intermediates) */
static inline float ndc2pix(float v, int S) { return (float)(fma((double)v + 1.0, (double)S, -1.0) * 0.5); }

/* auxiliary.h:46-56 */
static void get_rect(float px, float py, int max_radius, uint32_t gx, uint32_t gy, uint32_t *rmin, uint32_t *rmax)
{
    const float r = (float)max_radius;
    int v;
    v = f2i_rz((px - r) * 0.0625f); if (v < 0) v = 0; rmin[0] = (uint32_t)v < gx ? (uint32_t)v : gx;
    v = f2i_rz((py - r) * 0.0625f); if (v < 0) v = 0; rmin[1] = (uint32_t)v < gy ? (uint32_t)v : gy;
    v = f2i_rz((((px + r) + 16.0f) + -1.0f) * 0.0625f); if (v < 0) v = 0; rmax[0] = (uint32_t)v < gx ? (uint32_t)v : gx;
    v = f2i_rz((((py + r) + 16.0f) + -1.0f) * 0.0625f); if (v < 0) v = 0; rmax[1] = (uint32_t)v < gy ? (uint32_t)v : gy;
}

/* ---------------------------------------------------------------------------------------------
 * Stage 1: per-Gaussian preprocess (forward.cu:155-256) + inclusive scan (rasterizer_impl.cu:277).
 * Optional pointers (shs / colors_precomp / scales+rotations / cov3D_precomp) follow the
 * reference: NULL means absent.  Returns num_rendered.  All outputs are caller-allocated.
 * ------------------------------------------------------------------------------------------- */
int64_t oracle_preprocess(int P, int D, int M, const float *means3D, const float *scales, float scale_modifier,
                          const float *rotations, const float *opacities, const float *shs,
                          const float *cov3D_precomp, const float *colors_precomp, const float *viewmatrix,
                          const float *projmatrix, const float *campos, int W, int H, float tan_fovx,
                          float tan_fovy,
                          /* outputs */
                          int32_t *radii, float *means2D, float *depths, float *cov3Ds, float *rgb,
                          float *conic_opacity, uint8_t *clamped, uint32_t *tiles_touched,
                          uint32_t *point_offsets)
{
    const float focal_y = H / (2.0f * tan_fovy);
    const float focal_x = W / (2.0f * tan_fovx);
    const uint32_t gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    uint32_t running = 0;
    for (int i = 0; i < P; i++) {
        radii[i] = 0;
        tiles_touched[i] = 0;
        const float *m = means3D + 3 * i;
        do {
            const float depth = xf_row(viewmatrix, 2, m[0], m[1], m[2]);
            if (depth <= 0.2f) break; /* auxiliary.h:154 (also false for NaN -> kept, like the reference) */
            const float hx = xf_row(projmatrix, 0, m[0], m[1], m[2]);
            const float hy = xf_row(projmatrix, 1, m[0], m[1], m[2]);
            const float hw = xf_row(projmatrix, 3, m[0], m[1], m[2]);
            const float p_w = 1.0f / (hw + 0.0000001f);
            const float projx = hx * p_w, projy = hy * p_w;
            const float *c3;
            if (cov3D_precomp) c3 = cov3D_precomp + 6 * i;
            else {
                ref_cov3d(scales + 3 * i, scale_modifier, rotations + 4 * i, cov3Ds + 6 * i);
                c3 = cov3Ds + 6 * i;
            }
            float cov[3];
            ref_cov2d(m, focal_x, focal_y, tan_fovx, tan_fovy, c3, viewmatrix, cov);
            const float det = fmaf(cov[0], cov[2], -(cov[1] * cov[1]));
            if (det == 0.0f) break;
            const float det_inv = 1.0f / det;
            const float conic0 = cov[2] * det_inv, conic1 = cov[1] * (-det_inv), conic2 = cov[0] * det_inv;
            const float mid = (cov[0] + cov[2]) * 0.5f;
            const float s = sqrtf(fmaxf_(0.1f, fmaf(mid, mid, -det)));
            const float lmax = fmaxf_(mid + s, mid - s);
            const float my_radius = ceilf(3.0f * sqrtf(lmax));
            const int iradius = f2i_rz(my_radius);
            const float px = ndc2pix(projx, W), py = ndc2pix(projy, H);
            uint32_t rmin[2], rmax[2];
            get_rect(px, py, iradius, gx, gy, rmin, rmax);
            const uint32_t ntiles = (rmax[0] - rmin[0]) * (rmax[1] - rmin[1]);
            if (ntiles == 0) break;
            if (!colors_precomp) ref_sh_color(D, M, m, campos, shs + (size_t)i * M * 3, rgb + 3 * i, clamped + 3 * i);
            depths[i] = depth;
            radii[i] = iradius;
            means2D[2 * i] = px;
            means2D[2 * i + 1] = py;
            conic_opacity[4 * i] = conic0;
            conic_opacity[4 * i + 1] = conic1;
            conic_opacity[4 * i + 2] = conic2;
            conic_opacity[4 * i + 3] = opacities[i];
            tiles_touched[i] = ntiles;
        } while (0);
        running += tiles_touched[i];
        point_offsets[i] = running;
    }
    return (int64_t)running;
}

/* ---------------------------------------------------------------------------------------------
 * Stage 2: duplicateWithKeys + stable radix sort + identifyTileRanges
 * (rasterizer_impl.cu:70-138, 289-317).  keys/point_list sized num_rendered; ranges sized 2*T.
 * The reference sorts only bits [0, 32+bit); every tile id fits in `bit` bits so this equals a
 * full 64-bit stable sort.
 * ------------------------------------------------------------------------------------------- */
typedef struct { uint64_t key; uint32_t val; } kv_t;

static void merge_sort_kv(kv_t *a, kv_t *tmp, size_t n)
{
    for (size_t width = 1; width < n; width *= 2) {
        for (size_t lo = 0; lo < n; lo += 2 * width) {
            size_t mid = lo + width < n ? lo + width : n, hi = lo + 2 * width < n ? lo + 2 * width : n;
            size_t i = lo, j = mid, k = lo;
            while (i < mid && j < hi) tmp[k++] = (a[j].key < a[i].key) ? a[j++] : a[i++]; /* stable */
            while (i < mid) tmp[k++] = a[i++];
            while (j < hi) tmp[k++] = a[j++];
        }
        memcpy(a, tmp, n * sizeof(kv_t));
    }
}

void oracle_binning(int P, int W, int H, const int32_t *radii, const float *means2D, const float *depths,
                    const uint32_t *point_offsets, int64_t num_rendered,
                    /* outputs */
                    uint64_t *keys_sorted, uint32_t *point_list, uint32_t *ranges)
{
    const uint32_t gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)gx * gy);
    if (num_rendered <= 0) return;
    kv_t *kv = (kv_t *)malloc(sizeof(kv_t) * (size_t)num_rendered);
    kv_t *tmp = (kv_t *)malloc(sizeof(kv_t) * (size_t)num_rendered);
    for (int i = 0; i < P; i++) {
        if (radii[i] <= 0) continue;
        uint32_t off = (i == 0) ? 0 : point_offsets[i - 1];
        uint32_t rmin[2], rmax[2];
        get_rect(means2D[2 * i], means2D[2 * i + 1], radii[i], gx, gy, rmin, rmax);
        uint32_t dbits;
        memcpy(&dbits, depths + i, 4);
        for (uint32_t y = rmin[1]; y < rmax[1]; y++)
            for (uint32_t x = rmin[0]; x < rmax[0]; x++) {
                kv[off].key = ((uint64_t)(y * gx + x) << 32) | dbits;
                kv[off].val = (uint32_t)i;
                off++;
            }
    }
    merge_sort_kv(kv, tmp, (size_t)num_rendered);
    for (int64_t k = 0; k < num_rendered; k++) {
        keys_sorted[k] = kv[k].key;
        point_list[k] = kv[k].val;
    }
    for (int64_t k = 0; k < num_rendered; k++) {
        uint32_t cur = (uint32_t)(keys_sorted[k] >> 32);
        if (k == 0) ranges[2 * cur] = 0;
        else {
            uint32_t prev = (uint32_t)(keys_sorted[k - 1] >> 32);
            if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)k; ranges[2 * cur] = (uint32_t)k; }
        }
        if (k == num_rendered - 1) ranges[2 * cur + 1] = (uint32_t)num_rendered;
    }
    free(kv);
    free(tmp);
}

/* power exactly as compiled: fma(fma(dx, dx*a, dy*(dy*c)), -0.5, -(dy*(dx*b)))  (forward.cu:333-335) */
static inline float ref_power(float dx, float dy, float a, float b, float c)
{
    const float q = fmaf(dx, dx * a, dy * (dy * c));
    return fmaf(q, -0.5f, -(dy * (dx * b)));
}

/* ---------------------------------------------------------------------------------------------
 * Stage 3: per-tile front-to-back blend (forward.cu:261-374).  colors = colors_precomp or rgb.
 * ------------------------------------------------------------------------------------------- */
void oracle_render(int W, int H, const uint32_t *ranges, const uint32_t *point_list, const float *means2D,
                   const float *colors, const float *conic_opacity, const float *bg,
                   /* outputs */
                   float *final_T, uint32_t *n_contrib, float *out_color)
{
    const uint32_t gx = (W + TILE - 1) / TILE;
    for (int py = 0; py < H; py++)
        for (int px = 0; px < W; px++) {
            const uint32_t tile = (py / TILE) * gx + (px / TILE);
            const uint32_t lo = ranges[2 * tile], hi = ranges[2 * tile + 1];
            const float pxf = (float)px, pyf = (float)py;
            float T = 1.0f, C[3] = {0, 0, 0};
            uint32_t contributor = 0, last = 0;
            for (uint32_t k = lo; k < hi; k++) {
                contributor++;
                const uint32_t id = point_list[k];
                const float dx = means2D[2 * id] - pxf, dy = means2D[2 * id + 1] - pyf;
                const float *co = conic_opacity + 4 * id;
                const float power = ref_power(dx, dy, co[0], co[1], co[2]);
                if (power > 0.0f) continue;
                const float alpha = fminf_(0.99f, co[3] * expf(power));
                if (alpha < 1.0f / 255.0f) continue;
                const float test_T = T * (1.0f - alpha);
                if (test_T < 0.0001f) break; /* done */
                for (int ch = 0; ch < 3; ch++) C[ch] = fmaf(T, alpha * colors[3 * id + ch], C[ch]);
                T = test_T;
                last = contributor;
            }
            const size_t pix = (size_t)py * W + px;
            final_T[pix] = T;
            n_contrib[pix] = last;
            for (int ch = 0; ch < 3; ch++) out_color[(size_t)ch * H * W + pix] = fmaf(T, bg[ch], C[ch]);
        }
}

/* ---------------------------------------------------------------------------------------------
 * Stage 4: blend backward (backward.cu:399-557).  Per-pair terms in fp32 exactly as the reference
 * forms them; the cross-pixel sums (atomicAdd in the reference, order-nondeterministic) are
 * accumulated in double and rounded once.  Outputs sized: dL_dmean2D[3P], dL_dconic[4P],
 * dL_dopacity[P], dL_dcolors[3P] (zero-filled here).
 * ------------------------------------------------------------------------------------------- */
void oracle_render_backward(int P, int W, int H, const uint32_t *ranges, const uint32_t *point_list,
                            const float *bg, const float *means2D, const float *conic_opacity,
                            const float *colors, const float *final_Ts, const uint32_t *n_contrib,
                            const float *dL_dpixels,
                            /* outputs */
                            float *dL_dmean2D, float *dL_dconic, float *dL_dopacity, float *dL_dcolors)
{
    const uint32_t gx = (W + TILE - 1) / TILE;
    double *acc = (double *)calloc((size_t)P * 9, sizeof(double));
    const float ddelx_dx = (float)(0.5 * W), ddely_dy = (float)(0.5 * H);
    for (int py = 0; py < H; py++)
        for (int px = 0; px < W; px++) {
            const uint32_t tile = (py / TILE) * gx + (px / TILE);
            const uint32_t lo = ranges[2 * tile], hi = ranges[2 * tile + 1];
            const size_t pix = (size_t)py * W + px;
            const float pxf = (float)px, pyf = (float)py;
            const float T_final = final_Ts[pix];
            float T = T_final;
            const uint32_t last_contributor = n_contrib[pix];
            float accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0.0f, dpix[3];
            for (int ch = 0; ch < 3; ch++) dpix[ch] = dL_dpixels[(size_t)ch * H * W + pix];
            uint32_t contributor = hi - lo;
            for (uint32_t k = hi; k-- > lo;) {
                contributor--;
                if (contributor >= last_contributor) continue;
                const uint32_t id = point_list[k];
                const float dx = means2D[2 * id] - pxf, dy = means2D[2 * id + 1] - pyf;
                const float *co = conic_opacity + 4 * id;
                const float power = ref_power(dx, dy, co[0], co[1], co[2]);
                if (power > 0.0f) continue;
                const float G = expf(power);
                const float alpha = fminf_(0.99f, co[3] * G);
                if (alpha < 1.0f / 255.0f) continue;
                T = T / (1.0f - alpha);
                const float dchannel_dcolor = alpha * T;
                float dL_dalpha = 0.0f;
                double *a = acc + (size_t)id * 9;
                for (int ch = 0; ch < 3; ch++) {
                    const float c = colors[3 * id + ch];
                    accum_rec[ch] = fmaf(last_alpha, last_color[ch], (1.0f - last_alpha) * accum_rec[ch]);
                    last_color[ch] = c;
                    dL_dalpha = fmaf(c - accum_rec[ch], dpix[ch], dL_dalpha);
                    a[6 + ch] += (double)(dchannel_dcolor * dpix[ch]);
                }
                dL_dalpha *= T;
                last_alpha = alpha;
                float bg_dot = 0.0f;
                for (int ch = 0; ch < 3; ch++) bg_dot = fmaf(bg[ch], dpix[ch], bg_dot);
                dL_dalpha = fmaf(-T_final / (1.0f - alpha), bg_dot, dL_dalpha);
                const float dL_dG = co[3] * dL_dalpha;
                const float gdx = G * dx, gdy = G * dy;
                const float dG_ddelx = fmaf(-gdx, co[0], -(gdy * co[1]));
                const float dG_ddely = fmaf(-gdy, co[2], -(gdx * co[1]));
                a[0] += (double)(dL_dG * dG_ddelx * ddelx_dx);
                a[1] += (double)(dL_dG * dG_ddely * ddely_dy);
                a[2] += (double)(-0.5f * gdx * dx * dL_dG);
                a[3] += (double)(-0.5f * gdx * dy * dL_dG);
                a[4] += (double)(-0.5f * gdy * dy * dL_dG);
                a[5] += (double)(G * dL_dalpha);
            }
        }
    for (int i = 0; i < P; i++) {
        const double *a = acc + (size_t)i * 9;
        dL_dmean2D[3 * i] = (float)a[0];
        dL_dmean2D[3 * i + 1] = (float)a[1];
        dL_dmean2D[3 * i + 2] = 0.0f;
        dL_dconic[4 * i] = (float)a[2];
        dL_dconic[4 * i + 1] = (float)a[3];
        dL_dconic[4 * i + 2] = 0.0f;
        dL_dconic[4 * i + 3] = (float)a[4];
        dL_dopacity[i] = (float)a[5];
        dL_dcolors[3 * i] = (float)a[6];
        dL_dcolors[3 * i + 1] = (float)a[7];
        dL_dcolors[3 * i + 2] = (float)a[8];
    }
    free(acc);
}

/* ---------------------------------------------------------------------------------------------
 * Stage 5: per-Gaussian backward: computeCov2DCUDA (backward.cu:144-274), preprocessCUDA
 * (:346-396), SH backward (:20-139), cov3D backward (:278-341), dnormvdv (auxiliary.h:107-117).
 * cov3Ds = cov3D_precomp or the forward's cov3Ds.  Outputs must be zero-filled by the caller
 * (the reference returns torch::zeros tensors and only touches radii>0 rows).
 * ------------------------------------------------------------------------------------------- */
static void sh_backward(int deg, int M, const float *mean, const float *campos, const float *sh,
                        const uint8_t *clamped, const float *dL_dcolor, float *dL_dmean, float *dL_dsh)
{
    (void)M;
    const float ox = mean[0] - campos[0], oy = mean[1] - campos[1], oz = mean[2] - campos[2];
    const float len = sqrtf(fmaf(oz, oz, fmaf(ox, ox, oy * oy)));
    const float x = ox / len, y = oy / len, z = oz / len;
    float dRGB[3], dRGBdx[3] = {0, 0, 0}, dRGBdy[3] = {0, 0, 0}, dRGBdz[3] = {0, 0, 0};
    for (int c = 0; c < 3; c++) dRGB[c] = dL_dcolor[c] * (clamped[c] ? 0.0f : 1.0f);
#define SH(k, c) sh[(k) * 3 + (c)]
#define DSH(k, w) for (int c = 0; c < 3; c++) dL_dsh[(k) * 3 + c] = (w) * dRGB[c]
    DSH(0, SH_C0);
    if (deg > 0) {
        DSH(1, -SH_C1 * y);
        DSH(2, SH_C1 * z);
        DSH(3, -SH_C1 * x);
        for (int c = 0; c < 3; c++) {
            dRGBdx[c] = -SH_C1 * SH(3, c);
            dRGBdy[c] = -SH_C1 * SH(1, c);
            dRGBdz[c] = SH_C1 * SH(2, c);
        }
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            DSH(4, SH_C2[0] * xy);
            DSH(5, SH_C2[1] * yz);
            DSH(6, SH_C2[2] * (2.f * zz - xx - yy));
            DSH(7, SH_C2[3] * xz);
            DSH(8, SH_C2[4] * (xx - yy));
            for (int c = 0; c < 3; c++) {
                dRGBdx[c] += SH_C2[0] * y * SH(4, c) + SH_C2[2] * 2.f * -x * SH(6, c) + SH_C2[3] * z * SH(7, c) +
                             SH_C2[4] * 2.f * x * SH(8, c);
                dRGBdy[c] += SH_C2[0] * x * SH(4, c) + SH_C2[1] * z * SH(5, c) + SH_C2[2] * 2.f * -y * SH(6, c) +
                             SH_C2[4] * 2.f * -y * SH(8, c);
                dRGBdz[c] += SH_C2[1] * y * SH(5, c) + SH_C2[2] * 2.f * 2.f * z * SH(6, c) + SH_C2[3] * x * SH(7, c);
            }
            if (deg > 2) {
                DSH(9, SH_C3[0] * y * (3.f * xx - yy));
                DSH(10, SH_C3[1] * xy * z);
                DSH(11, SH_C3[2] * y * (4.f * zz - xx - yy));
                DSH(12, SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                DSH(13, SH_C3[4] * x * (4.f * zz - xx - yy));
                DSH(14, SH_C3[5] * z * (xx - yy));
                DSH(15, SH_C3[6] * x * (xx - 3.f * yy));
                for (int c = 0; c < 3; c++) {
                    dRGBdx[c] += (SH_C3[0] * SH(9, c) * 3.f * 2.f * xy + SH_C3[1] * SH(10, c) * yz +
                                  SH_C3[2] * SH(11, c) * -2.f * xy + SH_C3[3] * SH(12, c) * -3.f * 2.f * xz +
                                  SH_C3[4] * SH(13, c) * (-3.f * xx + 4.f * zz - yy) +
                                  SH_C3[5] * SH(14, c) * 2.f * xz + SH_C3[6] * SH(15, c) * 3.f * (xx - yy));
                    dRGBdy[c] += (SH_C3[0] * SH(9, c) * 3.f * (xx - yy) + SH_C3[1] * SH(10, c) * xz +
                                  SH_C3[2] * SH(11, c) * (-3.f * yy + 4.f * zz - xx) +
                                  SH_C3[3] * SH(12, c) * -3.f * 2.f * yz + SH_C3[4] * SH(13, c) * -2.f * xy +
                                  SH_C3[5] * SH(14, c) * -2.f * yz + SH_C3[6] * SH(15, c) * -3.f * 2.f * xy);
                    dRGBdz[c] += (SH_C3[1] * SH(10, c) * xy + SH_C3[2] * SH(11, c) * 4.f * 2.f * yz +
                                  SH_C3[3] * SH(12, c) * 3.f * (2.f * zz - xx - yy) +
                                  SH_C3[4] * SH(13, c) * 4.f * 2.f * xz + SH_C3[5] * SH(14, c) * (xx - yy));
                }
            }
        }
    }
#undef SH
#undef DSH
    const float ddx = dRGBdx[0] * dRGB[0] + dRGBdx[1] * dRGB[1] + dRGBdx[2] * dRGB[2];
    const float ddy = dRGBdy[0] * dRGB[0] + dRGBdy[1] * dRGB[1] + dRGBdy[2] * dRGB[2];
    const float ddz = dRGBdz[0] * dRGB[0] + dRGBdz[1] * dRGB[1] + dRGBdz[2] * dRGB[2];
    /* dnormvdv(float3) auxiliary.h:107-117 */
    const float sum2 = ox * ox + oy * oy + oz * oz;
    const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    dL_dmean[0] += ((+sum2 - ox * ox) * ddx - oy * ox * ddy - oz * ox * ddz) * invsum32;
    dL_dmean[1] += (-ox * oy * ddx + (sum2 - oy * oy) * ddy - oz * oy * ddz) * invsum32;
    dL_dmean[2] += (-ox * oz * ddx - oy * oz * ddy + (sum2 - oz * oz) * ddz) * invsum32;
}

static void cov3d_backward(const float *scale, float mod, const float *rot, const float *dL_dcov3D,
                           float *dL_dscale, float *dL_drot)
{
    const float r = rot[0], x = rot[1], y = rot[2], z = rot[3];
    /* R[col][row] as glm stores it (forward.cu:133-137 / backward.cu:288-292) */
    const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                           {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                           {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
    const float s[3] = {mod * scale[0], mod * scale[1], mod * scale[2]};
    /* M = S * R  =>  M[col][row] = s[row] * R[col][row] */
    float Mm[3][3], dS[3][3], dM[3][3];
    for (int c = 0; c < 3; c++)
        for (int w = 0; w < 3; w++) Mm[c][w] = s[w] * R[c][w];
    dS[0][0] = dL_dcov3D[0]; dS[0][1] = 0.5f * dL_dcov3D[1]; dS[0][2] = 0.5f * dL_dcov3D[2];
    dS[1][0] = 0.5f * dL_dcov3D[1]; dS[1][1] = dL_dcov3D[3]; dS[1][2] = 0.5f * dL_dcov3D[4];
    dS[2][0] = 0.5f * dL_dcov3D[2]; dS[2][1] = 0.5f * dL_dcov3D[4]; dS[2][2] = dL_dcov3D[5];
    /* dL_dM = 2 * M * dL_dSigma (column-major product: out[c][w] = sum_k A[k][w] * B[c][k]) */
    for (int c = 0; c < 3; c++)
        for (int w = 0; w < 3; w++)
            dM[c][w] = 2.0f * Mm[0][w] * dS[c][0] + 2.0f * Mm[1][w] * dS[c][1] + 2.0f * Mm[2][w] * dS[c][2];
    /* Rt = transpose(R), dMt = transpose(dM): Rt[c][w] = R[w][c] */
    float dMt[3][3];
    for (int c = 0; c < 3; c++)
        for (int w = 0; w < 3; w++) dMt[c][w] = dM[w][c];
    for (int k = 0; k < 3; k++)
        dL_dscale[k] = R[0][k] * dMt[k][0] + R[1][k] * dMt[k][1] + R[2][k] * dMt[k][2];
    for (int k = 0; k < 3; k++)
        for (int w = 0; w < 3; w++) dMt[k][w] *= s[k];
    dL_drot[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
    dL_drot[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) -
                 4 * x * (dMt[2][2] + dMt[1][1]);
    dL_drot[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) -
                 4 * y * (dMt[2][2] + dMt[0][0]);
    dL_drot[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) -
                 4 * z * (dMt[1][1] + dMt[0][0]);
}

void oracle_preprocess_backward(int P, int D, int M, const float *means3D, const int32_t *radii, const float *shs,
                                const uint8_t *clamped, const float *scales, const float *rotations,
                                float scale_modifier, const float *cov3Ds, const float *viewmatrix,
                                const float *projmatrix, int W, int H, float tan_fovx, float tan_fovy,
                                const float *campos, const float *dL_dmean2D, const float *dL_dconic,
                                const float *dL_dcolor,
                                /* outputs (caller zero-fills) */
                                float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh, float *dL_dscale,
                                float *dL_drot)
{
    const float h_y = H / (2.0f * tan_fovy);
    const float h_x = W / (2.0f * tan_fovx);
    const float *vm = viewmatrix, *proj = projmatrix;
    for (int i = 0; i < P; i++) {
        if (!(radii[i] > 0)) continue;
        const float *mean = means3D + 3 * i;
        const float *c3 = cov3Ds + 6 * i;
        /* ---- computeCov2DCUDA ---- */
        const float dcx = dL_dconic[4 * i], dcy = dL_dconic[4 * i + 1], dcz = dL_dconic[4 * i + 3];
        float t[3] = {xf_row(vm, 0, mean[0], mean[1], mean[2]), xf_row(vm, 1, mean[0], mean[1], mean[2]),
                      xf_row(vm, 2, mean[0], mean[1], mean[2])};
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float txtz = t[0] / t[2], tytz = t[1] / t[2];
        t[0] = fminf_(limx, fmaxf_(-limx, txtz)) * t[2];
        t[1] = fminf_(limy, fmaxf_(-limy, tytz)) * t[2];
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.0f : 1.0f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.0f : 1.0f;
        /* glm column-major: Mat[col][row] */
        const float J[3][3] = {{h_x / t[2], 0.0f, -(h_x * t[0]) / (t[2] * t[2])},
                               {0.0f, h_y / t[2], -(h_y * t[1]) / (t[2] * t[2])},
                               {0, 0, 0}};
        const float Wm[3][3] = {{vm[0], vm[4], vm[8]}, {vm[1], vm[5], vm[9]}, {vm[2], vm[6], vm[10]}};
        const float V[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
        float T[3][3], VtT[3][3], cov2D[3][3];
        for (int c = 0; c < 3; c++)
            for (int w = 0; w < 3; w++) T[c][w] = Wm[0][w] * J[c][0] + Wm[1][w] * J[c][1] + Wm[2][w] * J[c][2];
        /* transpose(Vrk) * T : A = V^T => A[k][w] = V[w][k] */
        for (int c = 0; c < 3; c++)
            for (int w = 0; w < 3; w++) VtT[c][w] = V[w][0] * T[c][0] + V[w][1] * T[c][1] + V[w][2] * T[c][2];
        /* transpose(T) * that : A[k][w] = T[w][k] */
        for (int c = 0; c < 3; c++)
            for (int w = 0; w < 3; w++) cov2D[c][w] = T[w][0] * VtT[c][0] + T[w][1] * VtT[c][1] + T[w][2] * VtT[c][2];
        const float a = cov2D[0][0] + 0.3f, b = cov2D[0][1], c = cov2D[1][1] + 0.3f;
        const float denom = a * c - b * b;
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float *dcov = dL_dcov3D + 6 * i;
        if (denom2inv != 0) {
            dL_da = denom2inv * (-c * c * dcx + 2 * b * c * dcy + (denom - a * c) * dcz);
            dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c) * dcx);
            dL_db = denom2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
            dcov[0] = (T[0][0] * T[0][0] * dL_da + T[0][0] * T[1][0] * dL_db + T[1][0] * T[1][0] * dL_dc);
            dcov[3] = (T[0][1] * T[0][1] * dL_da + T[0][1] * T[1][1] * dL_db + T[1][1] * T[1][1] * dL_dc);
            dcov[5] = (T[0][2] * T[0][2] * dL_da + T[0][2] * T[1][2] * dL_db + T[1][2] * T[1][2] * dL_dc);
            dcov[1] = 2 * T[0][0] * T[0][1] * dL_da + (T[0][0] * T[1][1] + T[0][1] * T[1][0]) * dL_db +
                      2 * T[1][0] * T[1][1] * dL_dc;
            dcov[2] = 2 * T[0][0] * T[0][2] * dL_da + (T[0][0] * T[1][2] + T[0][2] * T[1][0]) * dL_db +
                      2 * T[1][0] * T[1][2] * dL_dc;
            dcov[4] = 2 * T[0][2] * T[0][1] * dL_da + (T[0][1] * T[1][2] + T[0][2] * T[1][1]) * dL_db +
                      2 * T[1][1] * T[1][2] * dL_dc;
        } else {
            for (int k = 0; k < 6; k++) dcov[k] = 0;
        }
        const float dT00 = 2 * (T[0][0] * V[0][0] + T[0][1] * V[0][1] + T[0][2] * V[0][2]) * dL_da +
                           (T[1][0] * V[0][0] + T[1][1] * V[0][1] + T[1][2] * V[0][2]) * dL_db;
        const float dT01 = 2 * (T[0][0] * V[1][0] + T[0][1] * V[1][1] + T[0][2] * V[1][2]) * dL_da +
                           (T[1][0] * V[1][0] + T[1][1] * V[1][1] + T[1][2] * V[1][2]) * dL_db;
        const float dT02 = 2 * (T[0][0] * V[2][0] + T[0][1] * V[2][1] + T[0][2] * V[2][2]) * dL_da +
                           (T[1][0] * V[2][0] + T[1][1] * V[2][1] + T[1][2] * V[2][2]) * dL_db;
        const float dT10 = 2 * (T[1][0] * V[0][0] + T[1][1] * V[0][1] + T[1][2] * V[0][2]) * dL_dc +
                           (T[0][0] * V[0][0] + T[0][1] * V[0][1] + T[0][2] * V[0][2]) * dL_db;
        const float dT11 = 2 * (T[1][0] * V[1][0] + T[1][1] * V[1][1] + T[1][2] * V[1][2]) * dL_dc +
                           (T[0][0] * V[1][0] + T[0][1] * V[1][1] + T[0][2] * V[1][2]) * dL_db;
        const float dT12 = 2 * (T[1][0] * V[2][0] + T[1][1] * V[2][1] + T[1][2] * V[2][2]) * dL_dc +
                           (T[0][0] * V[2][0] + T[0][1] * V[2][1] + T[0][2] * V[2][2]) * dL_db;
        const float dJ00 = Wm[0][0] * dT00 + Wm[0][1] * dT01 + Wm[0][2] * dT02;
        const float dJ02 = Wm[2][0] * dT00 + Wm[2][1] * dT01 + Wm[2][2] * dT02;
        const float dJ11 = Wm[1][0] * dT10 + Wm[1][1] * dT11 + Wm[1][2] * dT12;
        const float dJ12 = Wm[2][0] * dT10 + Wm[2][1] * dT11 + Wm[2][2] * dT12;
        const float tz = 1.f / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        const float dtx = x_grad_mul * -h_x * tz2 * dJ02;
        const float dty = y_grad_mul * -h_y * tz2 * dJ12;
        const float dtz = -h_x * tz2 * dJ00 - h_y * tz2 * dJ11 + (2 * h_x * t[0]) * tz3 * dJ02 + (2 * h_y * t[1]) * tz3 * dJ12;
        float *dmean = dL_dmeans3D + 3 * i;
        /* transformVec4x3Transpose (auxiliary.h:89-97) */
        dmean[0] = vm[0] * dtx + vm[1] * dty + vm[2] * dtz;
        dmean[1] = vm[4] * dtx + vm[5] * dty + vm[6] * dtz;
        dmean[2] = vm[8] * dtx + vm[9] * dty + vm[10] * dtz;
        /* ---- preprocessCUDA (backward.cu:346-396) ---- */
        const float hw = xf_row(proj, 3, mean[0], mean[1], mean[2]);
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = (proj[0] * mean[0] + proj[4] * mean[1] + proj[8] * mean[2] + proj[12]) * m_w * m_w;
        const float mul2 = (proj[1] * mean[0] + proj[5] * mean[1] + proj[9] * mean[2] + proj[13]) * m_w * m_w;
        const float gx = dL_dmean2D[3 * i], gy = dL_dmean2D[3 * i + 1];
        dmean[0] += (proj[0] * m_w - proj[3] * mul1) * gx + (proj[1] * m_w - proj[3] * mul2) * gy;
        dmean[1] += (proj[4] * m_w - proj[7] * mul1) * gx + (proj[5] * m_w - proj[7] * mul2) * gy;
        dmean[2] += (proj[8] * m_w - proj[11] * mul1) * gx + (proj[9] * m_w - proj[11] * mul2) * gy;
        if (shs)
            sh_backward(D, M, mean, campos, shs + (size_t)i * M * 3, clamped + 3 * i, dL_dcolor + 3 * i, dmean,
                        dL_dsh + (size_t)i * M * 3);
        if (scales) cov3d_backward(scales + 3 * i, scale_modifier, rotations + 4 * i, dcov, dL_dscale + 3 * i, dL_drot + 4 * i);
    }
}

/* rasterizer_impl.cu:54-66 (markVisible) */
void oracle_mark_visible(int P, const float *means3D, const float *viewmatrix, const float *projmatrix,
                         uint8_t *present)
{
    (void)projmatrix;
    for (int i = 0; i < P; i++) {
        const float *m = means3D + 3 * i;
        const float depth = xf_row(viewmatrix, 2, m[0], m[1], m[2]);
        present[i] = !(depth <= 0.2f);
    }
}
