// sgr_meshlap.cu -- the refinement stage's mesh Laplacian smoothing regulariser, forward and backward.
//
// Replaces pytorch3d 0.7.4's mesh_laplacian_smoothing(surface_mesh, method) as sugar_trainers/refine.py:163-171,
// 778-780 can add it: every call builds a new Meshes, its sparse Laplacian L (the unique-edge table for "uniform", the
// cotangent weights of the moving vertices for "cot" / "cotcurv") and a sparse mm with its autograd.  The faces never
// change during refinement, so the vertex lists are built once (sugar_b200/meshloss.py: laplacian_topology, torch sort
// on the device) and what is left per step is, for y = the per-vertex rows and loss = sum_v |y_v| / V:
//
// Forward.  cot / cotcurv: one thread per face writes (cot_a, cot_b, cot_c, area) in pytorch3d's float32 operation
//   order (lap_face), so every vertex of a face reads the same bits.  Then one thread per vertex gathers its row over
//   its CSR list in ascending order -- uniform: the unique neighbours, a self-loop listed twice; cot / cotcurv: the
//   (face, corner) entries 3 f + k, each adding cot_prev x_next + cot_next x_prev, its row-sum share and its area,
//   which is L + L^T entry for entry, repeated vertices included -- and stores y with its row scale s (1 / deg,
//   norm_w, 0.25 inv_area) as a float4 for the backward.  |y_v| is summed per CTA in double and the CTA sums in a fixed
//   order by a second kernel (no float atomics: the result is identical from run to run).
// Backward, one thread per vertex, g_v = (g_loss / V) y_v / |y_v| (0 where |y_v| = 0), h = s g:
//   uniform  g_x = L^T g       = sum over the neighbour list of h_j - g_v
//   cot      g_x = L h - g                           (L symmetric: the same corner gather as the forward)
//   cotcurv  g_x = L h - rowsum(L) h
//   The upstream gradient is read on the device; the gathers run in ascending list order (deterministic).
//
// Numerics.  The face pass is float32, as pytorch3d's (Heron's formula is ill-conditioned on slivers there, in both);
// the gathers, row sums, norms and the reduction are in double.
#include <math.h>

#include "sgr_internal.cuh"
#include "sgr_reduce.cuh"

// The per-face and per-vertex arithmetic is plain C++: tests/test_meshlap_cpu.py compiles this file with
// -DSGR_MESHLAP_HOST_TEST and runs the same functions on the host against the oracle in float64.
#define SGR_HD __host__ __device__ __forceinline__

namespace sgr {

struct LapVec {
    double x, y, z;
};
SGR_HD LapVec operator+(LapVec a, LapVec b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
SGR_HD LapVec operator-(LapVec a, LapVec b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
SGR_HD LapVec operator*(double s, LapVec a) { return {s * a.x, s * a.y, s * a.z}; }
SGR_HD LapVec lap_vert(const float *__restrict__ verts, int i)
{
    const float *p = verts + 3 * (size_t)i;
    return {(double)p[0], (double)p[1], (double)p[2]};
}

// float32 products and sums never contracted into an FMA, as torch's elementwise kernels evaluate them
SGR_HD float lap_mul(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
SGR_HD float lap_add(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
SGR_HD float lap_sub(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
SGR_HD float lap_len(const float *p, const float *q)
{
    const float dx = lap_sub(p[0], q[0]), dy = lap_sub(p[1], q[1]), dz = lap_sub(p[2], q[2]);
    return sqrtf(lap_add(lap_add(lap_mul(dx, dx), lap_mul(dy, dy)), lap_mul(dz, dz)));
}

// cot_laplacian's per-face values in its float32 order: (cot_a, cot_b, cot_c) / 4 and the clamped Heron area
SGR_HD float4 lap_face(const float *__restrict__ verts, int i0, int i1, int i2)
{
    const float *v0 = verts + 3 * (size_t)i0, *v1 = verts + 3 * (size_t)i1, *v2 = verts + 3 * (size_t)i2;
    const float A = lap_len(v1, v2), B = lap_len(v0, v2), C = lap_len(v0, v1);
    const float s = lap_mul(0.5f, lap_add(lap_add(A, B), C));
    float q = lap_mul(lap_mul(lap_mul(s, lap_sub(s, A)), lap_sub(s, B)), lap_sub(s, C));
    q = q < 1e-12f ? 1e-12f : q;  // clamp_(min=eps): NaN stays NaN
    const float area = sqrtf(q);
    const float A2 = lap_mul(A, A), B2 = lap_mul(B, B), C2 = lap_mul(C, C);
    const float ca = lap_sub(lap_add(B2, C2), A2) / area;
    const float cb = lap_sub(lap_add(A2, C2), B2) / area;
    const float cc = lap_sub(lap_add(A2, B2), C2) / area;
    return make_float4(ca / 4.0f, cb / 4.0f, cc / 4.0f, area);
}

SGR_HD float lap_comp(float4 w, int k) { return k == 0 ? w.x : (k == 1 ? w.y : w.z); }

// One row of L applied to the vectors load(j), over vertex v's CSR list: lx = (L' load)_v with L' the off-diagonal part
// (uniform: unweighted, the caller scales by 1 / deg), rs its row sum, area the summed face areas (cot / cotcurv).
struct LapRow {
    LapVec lx;
    double rs, area;
};
template <class Load>
SGR_HD LapRow lap_gather(int method, int v, const int *__restrict__ faces, const float4 *__restrict__ face_w,
                         const int *__restrict__ ptr, const int *__restrict__ inc, Load load)
{
    LapRow r = {{0.0, 0.0, 0.0}, 0.0, 0.0};
    const int k0 = ptr[v], k1 = ptr[v + 1];
    if (method == SGR_MESH_LAP_UNIFORM) {
        for (int k = k0; k < k1; k++) r.lx = r.lx + load(inc[k]);
        r.rs = (double)(k1 - k0);
        return r;
    }
    for (int k = k0; k < k1; k++) {
        const int e = inc[k], f = e / 3, c = e - 3 * f;
        const int cn = c == 2 ? 0 : c + 1, cp = c == 0 ? 2 : c - 1;
        const float4 w = face_w[f];
        const double wn = lap_comp(w, cn), wp = lap_comp(w, cp);  // the cotangents opposite next and prev
        const int *fv = faces + 3 * (size_t)f;
        r.lx = r.lx + wp * load(fv[cn]) + wn * load(fv[cp]);
        r.rs += wn + wp;
        r.area += w.w;
    }
    return r;
}

// The forward's row of vertex v: y and its scale s (uniform 1 / deg, cot norm_w, cotcurv 0.25 inv_area)
SGR_HD LapVec lap_forward_row(int method, int v, const float *__restrict__ verts, const int *__restrict__ faces,
                              const float4 *__restrict__ face_w, const int *__restrict__ ptr,
                              const int *__restrict__ inc, double *scale)
{
    const LapRow r = lap_gather(method, v, faces, face_w, ptr, inc, [&](int j) { return lap_vert(verts, j); });
    const LapVec x = lap_vert(verts, v);
    if (method == SGR_MESH_LAP_UNIFORM) {
        const double s = r.rs > 0.0 ? 1.0 / r.rs : 0.0;
        *scale = s;
        return s * r.lx - x;
    }
    if (method == SGR_MESH_LAP_COT) {
        const double s = r.rs > 0.0 ? 1.0 / r.rs : r.rs;
        *scale = s;
        return s * r.lx - x;
    }
    const double s = 0.25 * (r.area > 0.0 ? 1.0 / r.area : 0.0);
    *scale = s;
    return s * (r.lx - r.rs * x);
}

// y / |y| from a stored row, 0 where y = 0
SGR_HD LapVec lap_unit(float4 q)
{
    const LapVec y = {(double)q.x, (double)q.y, (double)q.z};
    const double n = sqrt(y.x * y.x + y.y * y.y + y.z * y.z);
    return n > 0.0 ? (1.0 / n) * y : LapVec{0.0, 0.0, 0.0};
}

// The backward's row of vertex v from the forward's stored rows ys (y, s): dL/dx_v for an upstream factor c
SGR_HD LapVec lap_backward_row(int method, int v, const int *__restrict__ faces, const float4 *__restrict__ face_w,
                               const int *__restrict__ ptr, const int *__restrict__ inc,
                               const float4 *__restrict__ ys, double c)
{
    const LapRow r = lap_gather(method, v, faces, face_w, ptr, inc, [&](int j) {
        const float4 q = ys[j];
        return (double)q.w * lap_unit(q);
    });
    const float4 q = ys[v];
    const LapVec diag = method == SGR_MESH_LAP_COTCURV ? (r.rs * (double)q.w) * lap_unit(q) : lap_unit(q);
    return c * (r.lx - diag);
}

constexpr int LAP_THREADS = 256;

static int lap_blocks(int n) { return (n + LAP_THREADS - 1) / LAP_THREADS; }

__global__ void __launch_bounds__(LAP_THREADS) mesh_lap_face_kernel(int F, const float *__restrict__ verts,
                                                                     const int *__restrict__ faces,
                                                                     float4 *__restrict__ face_w)
{
    const int f = blockIdx.x * LAP_THREADS + threadIdx.x;
    if (f >= F) return;
    const int *fv = faces + 3 * (size_t)f;
    face_w[f] = lap_face(verts, __ldg(fv), __ldg(fv + 1), __ldg(fv + 2));
}

// grid-stride over the vertices; per CTA the sum of |y_v| in double
__global__ void __launch_bounds__(LAP_THREADS) mesh_lap_row_kernel(int method, int V, const float *__restrict__ verts,
                                                                    const int *__restrict__ faces,
                                                                    const float4 *__restrict__ face_w,
                                                                    const int *__restrict__ ptr,
                                                                    const int *__restrict__ inc, float4 *__restrict__ ys,
                                                                    double *__restrict__ partials)
{
    __shared__ double red[LAP_THREADS / 32];
    double t = 0.0;
    for (int v = blockIdx.x * LAP_THREADS + threadIdx.x; v < V; v += gridDim.x * LAP_THREADS) {
        double s;
        const LapVec y = lap_forward_row(method, v, verts, faces, face_w, ptr, inc, &s);
        ys[v] = make_float4((float)y.x, (float)y.y, (float)y.z, (float)s);
        t += sqrt(y.x * y.x + y.y * y.y + y.z * y.z);
    }
    const double s = cta_sum_by_warps<LAP_THREADS>(t, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(LAP_THREADS) mesh_lap_backward_kernel(int method, int V, double inv_v,
                                                                         const int *__restrict__ faces,
                                                                         const float4 *__restrict__ face_w,
                                                                         const int *__restrict__ ptr,
                                                                         const int *__restrict__ inc,
                                                                         const float4 *__restrict__ ys,
                                                                         const float *__restrict__ g_loss,
                                                                         float *__restrict__ g_verts)
{
    const int v = blockIdx.x * LAP_THREADS + threadIdx.x;
    if (v >= V) return;
    const LapVec g = lap_backward_row(method, v, faces, face_w, ptr, inc, ys, (double)__ldg(g_loss) * inv_v);
    g_verts[3 * (size_t)v] = (float)g.x;
    g_verts[3 * (size_t)v + 1] = (float)g.y;
    g_verts[3 * (size_t)v + 2] = (float)g.z;
}

static bool lap_args_ok(int32_t method, int32_t V, int32_t F, const char *who)
{
    if (method != SGR_MESH_LAP_UNIFORM && method != SGR_MESH_LAP_COT && method != SGR_MESH_LAP_COTCURV) {
        set_error("%s: unknown method %d (SGR_MESH_LAP_UNIFORM, _COT or _COTCURV)", who, method);
        return false;
    }
    if (V <= 0 || F <= 0 || F > INT32_MAX / 3) {
        set_error("%s: bad sizes V=%d F=%d (V > 0, 0 < F <= (2^31 - 1) / 3)", who, V, F);
        return false;
    }
    return true;
}

}  // namespace sgr

using namespace sgr;

#ifdef SGR_MESHLAP_HOST_TEST
// test-only build (never part of libsugar_b200.so): the face, row and backward functions looped on the host.
// norms[v] = |y_v| as the forward sums it; grads[v] = dL/dx_v for the upstream gradient g, before rounding to float.
extern "C" void mesh_lap_host(int method, int V, int F, const float *verts, const int *faces, const int *ptr,
                              const int *inc, double g, double *norms, double *grads)
{
    float4 *face_w = new float4[F > 0 ? F : 1];
    float4 *ys = new float4[V];
    if (method != SGR_MESH_LAP_UNIFORM)
        for (int f = 0; f < F; f++) face_w[f] = lap_face(verts, faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]);
    for (int v = 0; v < V; v++) {
        double s;
        const LapVec y = lap_forward_row(method, v, verts, faces, face_w, ptr, inc, &s);
        ys[v] = make_float4((float)y.x, (float)y.y, (float)y.z, (float)s);
        norms[v] = sqrt(y.x * y.x + y.y * y.y + y.z * y.z);
    }
    for (int v = 0; v < V; v++) {
        const LapVec d = lap_backward_row(method, v, faces, face_w, ptr, inc, ys, g / (double)V);
        grads[3 * v] = d.x;
        grads[3 * v + 1] = d.y;
        grads[3 * v + 2] = d.z;
    }
    delete[] face_w;
    delete[] ys;
}
#else
extern "C" {

int sgr_mesh_lap_forward(int32_t method, int32_t V, int32_t F, const float *verts, const int32_t *faces,
                         const int32_t *vert_ptr, const int32_t *vert_inc, float *face_w, float *vert_ys,
                         double *partials, float *loss, void *stream)
{
    if (!lap_args_ok(method, V, F, "sgr_mesh_lap_forward")) return SGR_EINVAL;
    const bool cot = method != SGR_MESH_LAP_UNIFORM;
    if (!verts || !vert_ptr || !vert_inc || !vert_ys || !partials || !loss || (cot && (!faces || !face_w))) {
        set_error("sgr_mesh_lap_forward: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (cot)
        SGR_LAUNCH(K_MISC, st,
                   mesh_lap_face_kernel<<<lap_blocks(F), LAP_THREADS, 0, st>>>(F, verts, faces, (float4 *)face_w));
    const int nb = lap_blocks(V) < SGR_MESH_LAP_PARTIALS ? lap_blocks(V) : SGR_MESH_LAP_PARTIALS;
    SGR_LAUNCH(K_MISC, st,
               mesh_lap_row_kernel<<<nb, LAP_THREADS, 0, st>>>(method, V, verts, faces, (const float4 *)face_w,
                                                                vert_ptr, vert_inc, (float4 *)vert_ys, partials));
    SGR_LAUNCH(K_MISC, st, sum_partials_kernel<1024><<<1, 1024, 0, st>>>(nb, 1.0 / (double)V, partials, loss));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_mesh_lap_backward(int32_t method, int32_t V, int32_t F, const int32_t *faces, const int32_t *vert_ptr,
                          const int32_t *vert_inc, const float *face_w, const float *vert_ys, const float *g_loss,
                          float *g_verts, void *stream)
{
    if (!lap_args_ok(method, V, F, "sgr_mesh_lap_backward")) return SGR_EINVAL;
    const bool cot = method != SGR_MESH_LAP_UNIFORM;
    if (!vert_ptr || !vert_inc || !vert_ys || !g_loss || !g_verts || (cot && (!faces || !face_w))) {
        set_error("sgr_mesh_lap_backward: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               mesh_lap_backward_kernel<<<lap_blocks(V), LAP_THREADS, 0, st>>>(
                   method, V, 1.0 / (double)V, faces, (const float4 *)face_w, vert_ptr, vert_inc,
                   (const float4 *)vert_ys, g_loss, g_verts));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
#endif  // SGR_MESHLAP_HOST_TEST
