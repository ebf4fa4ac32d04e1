// sgr_splatmesh.cu -- the level-set extraction's default depth source: every Gaussian as a view-facing "diamond" of
// two triangles, and a nearest-face triangle z-buffer over that mesh.
//
// Replaces, on the reference's default branch of compute_level_surface_points_from_camera_fast
// (use_gaussian_depth=False, sugar_scene/sugar_model.py:1880-1968):
//   SuGaR.splat_mesh(camera) with primitive 'diamond', triangle_scale 2, mode 'perspective' (:481-514, :695-728) and
//   pytorch3d 0.7.4's MeshRasterizer with blur_radius 0, read at faces_per_pixel index 0 (zbuf, pix_to_face).
//
// splat_mesh_kernel, one thread per Gaussian (reads 40 B, writes 48 B; the arithmetic is in double):
//   a0 = argmin(s) (lowest index on ties), a1 = (a0+1)%3, a2 = (a0+2)%3, R = quaternion_to_matrix(q) (two_s = 2/|q|^2);
//   vertices mu - t s_a1 R[:,a1], mu + t s_a2 R[:,a2], mu + t s_a1 R[:,a1], mu - t s_a2 R[:,a2] (t = triangle_scale);
//   in view space every vertex v moves along its own ray onto the plane through the centre c perpendicular to
//   d = c/|c|: v' = ((c.d)/(v.d)) v, with no guard at v.d <= 0 (as in the reference), then back to world space
//   through the inverse view matrix.
//
// Rasterizer, for any (verts [V,3], faces [F,3]) mesh:
//   mesh_setup_kernel     one thread per face: projects the three vertices (view z; projmatrix, / (w + 1e-7), the
//                         rasterizer's ndc2pix), drops the faces that can cover no pixel (a non-finite vertex, all
//                         z < 0, |area| <= pytorch3d's 1e-8 in its NDC units, an empty clipped box) and stores a
//                         64-byte record: the three barycentric planes relative to the box's corner, the view z's,
//                         the clipped pixel box and the face id; plus the box's count of 8x8-pixel pieces;
//   exclusive_scan        of the piece counts (sgr_scan.cu, three launches, 64-bit offsets);
//   mesh_fragment_kernel  grid-stride over the pieces, one thread per piece (at most 64 candidate pixels, so a
//                         background splat that covers half the image is spread over many threads): the piece's face by
//                         binary search over the offsets, the per-pixel test, and a 64-bit atomicMin of
//                         (float bits of pz << 32 | face) into a u64[H*W] key buffer preset to all ones;
//   mesh_resolve_kernel   one thread per pixel: zbuf f32 (-1 when empty), pix_to_face i64 (-1 when empty).
// A minimum over packed keys does not depend on the order of the atomics: the result is identical from run to run,
// and equal depths resolve to the lower face id.
//
// Per-pixel rule (pytorch3d's RasterizeMeshesNaive with perspective_correct, no culling, blur 0): with the sample
// point p of pixel (i, j) at ndc (2i+1)/S - 1 (pixel coordinate i in ndc2pix units) and b = bary(p),
// w_i = b_i z_j z_k, b' = w / max(sum w, 1e-8), pz = sum b'_i z_i; the face covers p iff every b'_i > 0 (i.e. every
// w_i > 0: the denominator is positive) and pz >= 0.  pytorch3d's +1e-8 on the area in the barycentrics scales all
// three alike and cancels in b' and pz; a covering pz that is not finite is dropped.
#include <math.h>

#include "sgr_internal.cuh"
#include "sgr_scan.cuh"

namespace sgr {

constexpr int SPM_THREADS = 256;
constexpr int PIECE = 8;              // pieces are PIECE x PIECE pixels of a face's clipped box

// row-vector transform p @ M[:3,:3] + M[3,:3] of a transposed 4x4 (the rasterizer's viewmatrix convention)
__device__ __forceinline__ double3 xf_point(const float *__restrict__ m, double x, double y, double z)
{
    return make_double3(x * m[0] + y * m[4] + z * m[8] + m[12], x * m[1] + y * m[5] + z * m[9] + m[13],
                        x * m[2] + y * m[6] + z * m[10] + m[14]);
}

__device__ __forceinline__ double dot3(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

__global__ void __launch_bounds__(SPM_THREADS) splat_mesh_kernel(int P, const float *__restrict__ points,
                                                                 const float *__restrict__ scaling,
                                                                 const float4 *__restrict__ quats,
                                                                 const float *__restrict__ view,
                                                                 const float *__restrict__ view_inv, float tri_scale,
                                                                 float4 *__restrict__ verts)
{
    __shared__ float m[32];  // view, view_inv
    if (threadIdx.x < 16) m[threadIdx.x] = view[threadIdx.x];
    else if (threadIdx.x < 32) m[threadIdx.x] = view_inv[threadIdx.x - 16];
    __syncthreads();
    const int g = blockIdx.x * SPM_THREADS + threadIdx.x;
    if (g >= P) return;
    const double mu[3] = {points[3 * (size_t)g], points[3 * (size_t)g + 1], points[3 * (size_t)g + 2]};
    const float s[3] = {scaling[3 * (size_t)g], scaling[3 * (size_t)g + 1], scaling[3 * (size_t)g + 2]};
    const float4 qf = __ldg(quats + g);
    int a0 = s[1] < s[0] ? 1 : 0;
    if (s[2] < (a0 ? s[1] : s[0])) a0 = 2;
    const int a1 = a0 == 2 ? 0 : a0 + 1, a2 = a0 == 0 ? 2 : a0 - 1;
    // pytorch3d quaternion_to_matrix (real part first)
    const double r = qf.x, i = qf.y, j = qf.z, k = qf.w;
    const double two_s = 2.0 / (r * r + i * i + j * j + k * k);
    const double3 col0 = make_double3(1.0 - two_s * (j * j + k * k), two_s * (i * j + k * r), two_s * (i * k - j * r));
    const double3 col1 = make_double3(two_s * (i * j - k * r), 1.0 - two_s * (i * i + k * k), two_s * (j * k + i * r));
    const double3 col2 = make_double3(two_s * (i * k + j * r), two_s * (j * k - i * r), 1.0 - two_s * (i * i + j * j));
    // selects, not indexed arrays: a runtime index would put R and s in local memory
    const double3 c1 = a1 == 0 ? col0 : (a1 == 1 ? col1 : col2), c2 = a2 == 0 ? col0 : (a2 == 1 ? col1 : col2);
    const double t1 = (double)tri_scale * (a1 == 0 ? s[0] : (a1 == 1 ? s[1] : s[2]));
    const double t2 = (double)tri_scale * (a2 == 0 ? s[0] : (a2 == 1 ? s[1] : s[2]));
    const double e1[3] = {t1 * c1.x, t1 * c1.y, t1 * c1.z};
    const double e2[3] = {t2 * c2.x, t2 * c2.y, t2 * c2.z};
    // diamond (0,-1,0), (0,0,1), (0,1,0), (0,0,-1) in the permuted frame
    const double sy[4] = {-1.0, 0.0, 1.0, 0.0}, sz[4] = {0.0, 1.0, 0.0, -1.0};
    const double3 c = xf_point(m, mu[0], mu[1], mu[2]);
    const double inv_len = 1.0 / fmax(sqrt(dot3(c, c)), 1e-12);  // torch.nn.functional.normalize
    const double3 d = make_double3(c.x * inv_len, c.y * inv_len, c.z * inv_len);
    const double pc = dot3(c, d);
    float o[12];
#pragma unroll
    for (int v = 0; v < 4; v++) {
        const double3 vv = xf_point(m, mu[0] + sy[v] * e1[0] + sz[v] * e2[0], mu[1] + sy[v] * e1[1] + sz[v] * e2[1],
                                    mu[2] + sy[v] * e1[2] + sz[v] * e2[2]);
        const double f = pc / dot3(vv, d);
        const double3 w = xf_point(m + 16, f * vv.x, f * vv.y, f * vv.z);
        o[3 * v] = (float)w.x;
        o[3 * v + 1] = (float)w.y;
        o[3 * v + 2] = (float)w.z;
    }
    float4 *out = verts + 3 * (size_t)g;
    out[0] = make_float4(o[0], o[1], o[2], o[3]);
    out[1] = make_float4(o[4], o[5], o[6], o[7]);
    out[2] = make_float4(o[8], o[9], o[10], o[11]);
}

// Face record (64 B): planes b_i(x, y) = A_i dx + B_i dy + C_i with (dx, dy) = pixel - box corner,
//   r0 = (A0, B0, C0, A1)  r1 = (B1, C1, A2, B2)  r2 = (C2, z0, z1, z2)  r3 = (x0 | y0 << 16, bw | bh << 16, face, nx)
struct FaceSetup {
    float4 r0, r1, r2, r3;
};

__global__ void __launch_bounds__(SPM_THREADS) mesh_setup_kernel(int F, int V, const float *__restrict__ verts,
                                                                 const long long *__restrict__ faces,
                                                                 const float *__restrict__ view,
                                                                 const float *__restrict__ proj, int W, int H,
                                                                 double area_eps, FaceSetup *__restrict__ rec,
                                                                 unsigned *__restrict__ npieces)
{
    __shared__ float m[32];  // view, proj
    if (threadIdx.x < 16) m[threadIdx.x] = view[threadIdx.x];
    else if (threadIdx.x < 32) m[threadIdx.x] = proj[threadIdx.x - 16];
    __syncthreads();
    const int f = blockIdx.x * SPM_THREADS + threadIdx.x;
    if (f >= F) return;
    double x[3], y[3], z[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const long long id = __ldg(faces + 3 * (size_t)f + c);
        ok = ok && id >= 0 && id < V;
        const long long vi = ok ? id : 0;
        const double px = verts[3 * vi], py = verts[3 * vi + 1], pz = verts[3 * vi + 2];
        z[c] = px * m[2] + py * m[6] + pz * m[10] + m[14];
        const double hx = px * m[16] + py * m[20] + pz * m[24] + m[28];
        const double hy = px * m[17] + py * m[21] + pz * m[25] + m[29];
        const double hw = px * m[19] + py * m[23] + pz * m[27] + m[31];
        const double inv_w = __drcp_rn(hw + 1e-7);
        x[c] = ((hx * inv_w + 1.0) * W - 1.0) * 0.5;  // ndc2pix
        y[c] = ((hy * inv_w + 1.0) * H - 1.0) * 0.5;
        ok = ok && isfinite(x[c]) && isfinite(y[c]) && isfinite(z[c]);
    }
    unsigned n = 0;
    if (ok && fmax(fmax(z[0], z[1]), z[2]) >= 0.0) {
        const double area = (x[2] - x[0]) * (y[1] - y[0]) - (y[2] - y[0]) * (x[1] - x[0]);
        const double xmin = fmin(fmin(x[0], x[1]), x[2]), xmax = fmax(fmax(x[0], x[1]), x[2]);
        const double ymin = fmin(fmin(y[0], y[1]), y[2]), ymax = fmax(fmax(y[0], y[1]), y[2]);
        const int x0 = (int)ceil(fmax(xmin, 0.0)), x1 = (int)floor(fmin(xmax, (double)(W - 1)));
        const int y0 = (int)ceil(fmax(ymin, 0.0)), y1 = (int)floor(fmin(ymax, (double)(H - 1)));
        if (fabs(area) > area_eps && x0 <= x1 && y0 <= y1) {
            const int bw = x1 - x0 + 1, bh = y1 - y0 + 1;
            const int nx = (bw + PIECE - 1) / PIECE;
            n = (unsigned)nx * (unsigned)((bh + PIECE - 1) / PIECE);
            // b_i = E(p, a, b) / area over the edges (v1, v2), (v2, v0), (v0, v1); E(p, a, b) =
            // (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x), taken relative to the box corner (x0, y0)
            const double inv_area = __drcp_rn(area);
            float pl[9];
#pragma unroll
            for (int e = 0; e < 3; e++) {
                const int a = (e + 1) % 3, b = (e + 2) % 3;
                const double ey = y[b] - y[a], ex = x[b] - x[a];
                pl[3 * e] = (float)(ey * inv_area);
                pl[3 * e + 1] = (float)(-ex * inv_area);
                pl[3 * e + 2] = (float)(((x0 - x[a]) * ey - (y0 - y[a]) * ex) * inv_area);
            }
            FaceSetup r;
            r.r0 = make_float4(pl[0], pl[1], pl[2], pl[3]);
            r.r1 = make_float4(pl[4], pl[5], pl[6], pl[7]);
            r.r2 = make_float4(pl[8], (float)z[0], (float)z[1], (float)z[2]);
            r.r3 = make_float4(__uint_as_float((unsigned)x0 | ((unsigned)y0 << 16)),
                               __uint_as_float((unsigned)bw | ((unsigned)bh << 16)), __int_as_float(f),
                               __int_as_float(nx));
            rec[f] = r;
        }
    }
    npieces[f] = n;
    if (f == 0) npieces[F] = 0;
}

__global__ void __launch_bounds__(SPM_THREADS) mesh_fragment_kernel(int F, int W, const unsigned long long *__restrict__ off,
                                                                    const FaceSetup *__restrict__ rec,
                                                                    unsigned long long *__restrict__ keys)
{
    const unsigned long long total = off[F];
    const unsigned long long stride = (unsigned long long)gridDim.x * SPM_THREADS;
    for (unsigned long long p = (unsigned long long)blockIdx.x * SPM_THREADS + threadIdx.x; p < total; p += stride) {
        int lo = 0, hi = F;  // off[lo] <= p < off[hi]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(off + mid) <= p) lo = mid;
            else hi = mid;
        }
        const FaceSetup r = rec[lo];
        const unsigned corner = __float_as_uint(r.r3.x), size = __float_as_uint(r.r3.y);
        const int face = __float_as_int(r.r3.z), nx = __float_as_int(r.r3.w);
        const int piece = (int)(p - __ldg(off + lo));
        const int dx0 = PIECE * (piece % nx), dy0 = PIECE * (piece / nx);
        const int x0 = corner & 0xffff, y0 = corner >> 16;
        const int ex = min(PIECE, (int)(size & 0xffff) - dx0), ey = min(PIECE, (int)(size >> 16) - dy0);
        const float z0 = r.r2.y, z1 = r.r2.z, z2 = r.r2.w;
        const float zz0 = z1 * z2, zz1 = z0 * z2, zz2 = z0 * z1;
        for (int yy = 0; yy < ey; yy++) {
            const float dy = (float)(dy0 + yy);
            const float c0 = fmaf(r.r0.y, dy, r.r0.z), c1 = fmaf(r.r1.x, dy, r.r1.y), c2 = fmaf(r.r1.w, dy, r.r2.x);
            unsigned long long *row = keys + (size_t)(y0 + dy0 + yy) * W + x0 + dx0;
            for (int xx = 0; xx < ex; xx++) {
                const float dx = (float)(dx0 + xx);
                const float w0 = fmaf(r.r0.x, dx, c0) * zz0, w1 = fmaf(r.r0.w, dx, c1) * zz1,
                            w2 = fmaf(r.r1.z, dx, c2) * zz2;
                if (!(w0 > 0.0f && w1 > 0.0f && w2 > 0.0f)) continue;
                float pz = (w0 * z0 + w1 * z1 + w2 * z2) / fmaxf(w0 + w1 + w2, 1e-8f);
                if (!(pz >= 0.0f && pz <= 3.402823466e38f)) continue;
                if (pz == 0.0f) pz = 0.0f;  // -0.0 packs as the largest key
                const unsigned long long key = ((unsigned long long)__float_as_uint(pz) << 32) | (unsigned)face;
                // keys only decrease: a stale read can only be larger, so skipping on it is safe
                if (key < row[xx]) atomicMin(row + xx, key);
            }
        }
    }
}

__global__ void __launch_bounds__(SPM_THREADS) mesh_resolve_kernel(int n, const unsigned long long *__restrict__ keys,
                                                                   float *__restrict__ zbuf,
                                                                   long long *__restrict__ pix_to_face)
{
    const int i = blockIdx.x * SPM_THREADS + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = keys[i];
    const bool empty = k == ~0ull;
    zbuf[i] = empty ? -1.0f : __uint_as_float((unsigned)(k >> 32));
    pix_to_face[i] = empty ? -1ll : (long long)(unsigned)(k & 0xffffffffu);
}

static int spm_blocks(long long n, int threads) { return (int)((n + threads - 1) / threads); }

struct RasterScratch {
    FaceSetup *rec;
    unsigned *npieces;
    unsigned long long *off, *block_sums, *keys;
    static RasterScratch carve(Layout &l, int F, int W, int H)
    {
        RasterScratch s;
        s.rec = l.take<FaceSetup>(F);
        s.npieces = l.take<unsigned>((size_t)F + 1);  // a zero count past the last face: off[F] is the total
        s.off = l.take<unsigned long long>((size_t)F + 1);
        s.block_sums = l.take<unsigned long long>(scan_block_sums((size_t)F + 1));
        s.keys = l.take<unsigned long long>((size_t)W * H);
        return s;
    }
};

// the packed key keeps the face id in 32 bits: F <= 2^31 - 1 by its type, so ~0 never names a face
static bool raster_sizes_ok(int F, int W, int H)
{
    return F >= 0 && W >= 0 && H >= 0 && W <= 65535 && H <= 65535 && (long long)W * H <= INT32_MAX;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_splat_mesh(int32_t P, const float *points, const float *scaling, const float *quaternions,
                   const float *viewmatrix, const float *view_inverse, float triangle_scale, float *verts, void *stream)
{
    if (P < 0 || P > INT32_MAX / 4) {
        set_error("sgr_splat_mesh: bad size P=%d (0 <= P <= (2^31 - 1) / 4)", P);
        return SGR_EINVAL;
    }
    if (P == 0) return SGR_OK;
    if (!points || !scaling || !quaternions || !viewmatrix || !view_inverse || !verts) {
        set_error("sgr_splat_mesh: null pointer");
        return SGR_EINVAL;
    }
    if (((size_t)quaternions | (size_t)verts) & 15) {
        set_error("sgr_splat_mesh: quaternions and verts must be 16-byte aligned");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               splat_mesh_kernel<<<spm_blocks(P, SPM_THREADS), SPM_THREADS, 0, st>>>(
                   P, points, scaling, (const float4 *)quaternions, viewmatrix, view_inverse, triangle_scale,
                   (float4 *)verts));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

size_t sgr_mesh_raster_scratch_bytes(int32_t F, int32_t W, int32_t H)
{
    return raster_sizes_ok(F, W, H) ? layout_bytes([&](Layout &l) { RasterScratch::carve(l, F, W, H); }) : 0;
}

int sgr_mesh_raster(int32_t V, int32_t F, const float *verts, const int64_t *faces, const float *viewmatrix,
                    const float *projmatrix, int32_t W, int32_t H, float *zbuf, int64_t *pix_to_face, void *scratch,
                    void *stream)
{
    if (V < 0 || !raster_sizes_ok(F, W, H)) {
        set_error("sgr_mesh_raster: bad sizes V=%d F=%d W=%d H=%d (W, H <= 65535, W*H <= 2^31 - 1)", V, F, W, H);
        return SGR_EINVAL;
    }
    const long long n_pix = (long long)W * H;
    if (n_pix == 0) return SGR_OK;
    if (!zbuf || !pix_to_face || !scratch || (F > 0 && (!verts || !faces || !viewmatrix || !projmatrix))) {
        set_error("sgr_mesh_raster: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    const RasterScratch s = RasterScratch::carve(l, F, W, H);
    SGR_CUDA(cudaMemsetAsync(s.keys, 0xff, (size_t)n_pix * 8, st));
    if (F > 0) {
        // pytorch3d drops |area| <= 1e-8 in its NDC units, 2 / min(W, H) per pixel
        const double half = 0.5 * (double)(W < H ? W : H);
        const double area_eps = 1e-8 * half * half;
        SGR_LAUNCH(K_MISC, st,
                   mesh_setup_kernel<<<spm_blocks(F, SPM_THREADS), SPM_THREADS, 0, st>>>(
                       F, V, verts, (const long long *)faces, viewmatrix, projmatrix, W, H, area_eps, s.rec, s.npieces));
        exclusive_scan(K_MISC, (size_t)F + 1, s.npieces, s.off, s.block_sums, s.off, st);
        SGR_LAUNCH(K_MISC, st,
                   mesh_fragment_kernel<<<device_sm_count() * 8, SPM_THREADS, 0, st>>>(F, W, s.off, s.rec, s.keys));
    }
    SGR_LAUNCH(K_MISC, st,
               mesh_resolve_kernel<<<spm_blocks(n_pix, SPM_THREADS), SPM_THREADS, 0, st>>>(
                   (int)n_pix, s.keys, zbuf, (long long *)pix_to_face));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
