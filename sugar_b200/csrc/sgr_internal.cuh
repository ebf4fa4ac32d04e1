// sgr_internal.cuh -- shared declarations of libsugar_b200 (sm_90a only).
//
// Layout of the three opaque round-trip buffers (the reference's GeometryState / BinningState /
// ImageState, rasterizer_impl.h:30-63, are opaque to Python so the layout is ours):
//
//   geometry (per Gaussian)            image (per pixel / per tile)          binning (per instance)
//   rec    float4[3P]  48 B splat rec  final_T  f32[HW]                      inst_a  u64[C] depth|idx
//   rect   ushort4[P]   8 B tile rect  n_contrib u32[HW]                     inst_b  u64[C] sort pong
//   depth  f32[P]       4 B            tile_count u32[T]  tile_start u32[T+1] (plist is laid out FIRST)
//   sh_jac f32[9P]     36 B            tile_cursor u32[T] tile_order u32[T] counters u32[16]
//
// Splat record (what the blend kernels gather, 48 B = 1.5 sectors instead of the reference's
// three separate gathers xy / conic_opacity / rgb = 3-4 sectors):
//   rec[0] = (x, y, conic_a, conic_b)   rec[1] = (conic_c, tau, opacity, r)   rec[2] = (g, b, clamp bits, id)
// tau = conservative power threshold below which alpha < 1/255 is certain (see blend kernels).
// sh_jac = the SH colour's derivatives by the normalised view direction, three RGB triples per Gaussian
// (dRGBdx, dRGBdy, dRGBdz of backward.cu:36-128): the backward's view-direction term of dL/dmean3D needs only
// these, so it never reads the SH coefficients.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sugar_b200.h"

#define SGR_TILE 16
#define SGR_ALIGN 256

namespace sgr {

static inline size_t align_up(size_t v, size_t a = SGR_ALIGN) { return (v + a - 1) / a * a; }

// Walks one buffer's layout.  Started at the buffer's base it hands out the arrays in order, each SGR_ALIGN-aligned;
// started at null it only measures.  Every layout is one function over a Layout, called both to size the buffer and
// to carve it, so the size a caller allocates and the arrays the kernels write cannot disagree.
class Layout {
  public:
    explicit Layout(const void *base = nullptr) : start_(align_up((size_t)base)), at_(start_) {}
    template <class T> T *take(size_t n)
    {
        T *p = (T *)at_;
        at_ += align_up(n * sizeof(T));
        return p;
    }
    // the bytes to allocate: what the walk consumed, plus the slack that aligns an unaligned base
    size_t bytes() const { return at_ - start_ + SGR_ALIGN; }

  private:
    size_t start_, at_;
};

// the size of the layout `walk` takes from a Layout
template <class Walk> size_t layout_bytes(Walk walk)
{
    Layout l;
    walk(l);
    return l.bytes();
}

struct GeomState {
    float4 *rec;
    ushort4 *rect;
    float *depth;
    float *sh_jac;  // [P][9] (dRGB/dx, dRGB/dy, dRGB/dz) of the SH colour; zero rows for culled Gaussians
    static GeomState carve(Layout &l, size_t P)
    {
        GeomState s;
        s.rec = l.take<float4>(3 * P);
        s.rect = l.take<ushort4>(P);
        s.depth = l.take<float>(P);
        s.sh_jac = l.take<float>(9 * P);
        return s;
    }
};

struct ImageState {
    float *final_T;
    uint32_t *n_contrib;
    uint32_t *tile_count;
    uint32_t *tile_start;  // T+1
    uint32_t *tile_cursor;  // after scatter: the end of each tile's live list [tile_start[t], tile_cursor[t])
    uint32_t *tile_order;  // tiles by decreasing instance count: launch order of the blend kernels
    uint32_t *counters;    // [0] = num_rendered, [1] = overflow flag
    static ImageState carve(Layout &l, size_t W, size_t H)
    {
        const size_t T = ((W + 15) / 16) * ((H + 15) / 16);
        ImageState s;
        s.final_T = l.take<float>(W * H);
        s.n_contrib = l.take<uint32_t>(W * H);
        s.tile_count = l.take<uint32_t>(T);
        s.tile_start = l.take<uint32_t>(T + 1);
        s.tile_cursor = l.take<uint32_t>(T);
        s.tile_order = l.take<uint32_t>(T);
        s.counters = l.take<uint32_t>(16);
        return s;
    }
};

struct BinState {
    // plist comes first so that its address does not depend on the capacity the forward chose
    // (backward and inspection only know num_rendered, not the optimistic capacity).
    uint32_t *plist;
    uint64_t *inst_a;
    uint64_t *inst_b;
    static BinState carve(Layout &l, size_t C)
    {
        if (C == 0) C = 1;
        BinState s;
        s.plist = l.take<uint32_t>(C);
        s.inst_a = l.take<uint64_t>(C);
        s.inst_b = l.take<uint64_t>(C);
        return s;
    }
};

// the backward's blend accumulators, 32 B per Gaussian
static inline float *carve_grad_acc(Layout &l, size_t P) { return l.take<float>(8 * P); }

// Per-view constants passed by value (constant bank).  The matrices, camera position and background stay device
// pointers, as in the reference API: kernels load them through the read-only path (16+16+3+3 floats, L1-resident).
struct ViewConsts {
    const float *viewmatrix;
    const float *projmatrix;
    const float *campos;
    const float *bg;
    int W, H, gx, gy;
    float tanfovx, tanfovy, focal_x, focal_y, scale_modifier;
    int D, M;
    int prefiltered;
};

static inline ViewConsts view_consts(const SgrView *view, int M)
{
    ViewConsts v;
    v.viewmatrix = view->viewmatrix;
    v.projmatrix = view->projmatrix;
    v.campos = view->campos;
    v.bg = view->bg;
    v.W = view->image_width;
    v.H = view->image_height;
    v.gx = (v.W + SGR_TILE - 1) / SGR_TILE;
    v.gy = (v.H + SGR_TILE - 1) / SGR_TILE;
    v.tanfovx = view->tanfovx;
    v.tanfovy = view->tanfovy;
    v.focal_y = v.H / (2.0f * view->tanfovy);  // rasterizer_impl.cu:222-223
    v.focal_x = v.W / (2.0f * view->tanfovx);
    v.scale_modifier = view->scale_modifier;
    v.D = view->sh_degree;
    v.M = M;
    v.prefiltered = view->prefiltered;
    return v;
}

static inline bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);
int device_sm_count();  // SMs of the current device (grid sizes of the grid-stride kernels)

// Per-device host state (slot pools, one-time set-up, events) is kept in tables of SGR_MAX_DEVICES entries.
#define SGR_MAX_DEVICES 64
int current_device(int *dev);  // the current device, or SGR_EINVAL if it is beyond SGR_MAX_DEVICES
// One-time set-up per device, e.g. opting a kernel in to > 48 KB of dynamic shared memory (the call is not free).
// once_per_device runs init() under a lock the first time it is called with `once` on the current device; calls may
// come from several threads (autograd engine threads of different devices).  A failed init() is retried next time.
struct DeviceOnce {
    bool done[SGR_MAX_DEVICES];
};
int once_per_device(DeviceOnce &once, int (*init)());

// Kernel bookkeeping: every launch of one of OUR kernels goes through SGR_LAUNCH so that
// sgr_launch_count() is a measured number and, when profiling is switched on, each launch is
// bracketed by CUDA events on the launching stream (bench.py reads the per-kernel durations).
enum KernelKind {
    K_PREPROCESS = 0, K_TILE_SCAN, K_SCATTER, K_SORT_SMEM, K_SORT_GLOBAL, K_BLEND_FWD, K_BLEND_BWD, K_PRE_BWD,
    K_FIELD_PACK, K_FIELD_FWD, K_FIELD_BWD, K_FIELD_UNPACK, K_KNN, K_KNN_QUERY, K_MISC, K_FINALIZE, K_PEER_REDUCE,
    K_PEER_SYNC, K_LOSS_FWD, K_LOSS_BWD, K_DENSEST_FWD, K_DENSEST_BWD, K_MESH_NC_FWD, K_MESH_NC_BWD, K_NUM_KINDS
};
void prof_begin(int kind, cudaStream_t st);
void prof_end(cudaStream_t st);
void note_launches(int extra);  // launches not individually bracketed by prof_begin
#define SGR_LAUNCH(kind, st, ...)     \
    do {                              \
        sgr::prof_begin((kind), (st)); \
        __VA_ARGS__;                  \
        sgr::prof_end((st));          \
    } while (0)

#define SGR_CUDA(call)                                            \
    do {                                                          \
        cudaError_t e__ = (call);                                 \
        if (e__ != cudaSuccess) return sgr::cuda_fail(e__, #call); \
    } while (0)

// ---------------------------------------------------------------------------------------------
// Device math shared by forward and backward.  The "exact" helpers spell out every rounding
// with _rn intrinsics (never re-fused by ptxas) in the order nvcc 12.9 emits for the reference
// sources, so depth / pixel position / radius / tile rect are bit-identical to the reference
// build (DESIGN.md "Bit-exact chain").
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__

// m[r]*x + m[4+r]*y + m[8+r]*z + m[12+r]   (auxiliary.h:58-77)
__device__ __forceinline__ float xf_row(const float *__restrict__ m, int r, float x, float y, float z)
{
    float t = __fmul_rn(y, m[4 + r]);
    t = __fmaf_rn(x, m[r], t);
    t = __fmaf_rn(z, m[8 + r], t);
    return __fadd_rn(t, m[12 + r]);
}

// Sigma = (S R)^T (S R) from scale + quaternion (forward.cu:118-152)
__device__ __forceinline__ void cov3d_from_scale_rot(float s0, float s1, float s2, float mod, float4 q, float *cov)
{
    const float sx = __fmul_rn(mod, s0), sy = __fmul_rn(mod, s1), sz = __fmul_rn(mod, s2);
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float rz = __fmul_rn(r, z), xz = __fmul_rn(x, z), rx = __fmul_rn(r, x);
    const float yy_zz = __fadd_rn(yy, zz);
    const float xy_m_rz = __fmaf_rn(x, y, -rz);
    const float xy_p_rz = __fmaf_rn(x, y, rz);
    const float ry_p_xz = __fmaf_rn(r, y, xz);
    const float xz_m_ry = __fmaf_rn(-r, y, xz);
    const float yz_m_rx = __fmaf_rn(y, z, -rx);
    const float yz_p_rx = __fmaf_rn(y, z, rx);
    const float xx_zz = __fmaf_rn(x, x, zz);
    const float xx_yy = __fmaf_rn(x, x, yy);
    const float R00 = __fsub_rn(1.0f, __fadd_rn(yy_zz, yy_zz));
    const float R01 = __fadd_rn(xy_m_rz, xy_m_rz);
    const float R02 = __fadd_rn(ry_p_xz, ry_p_xz);
    const float R10 = __fadd_rn(xy_p_rz, xy_p_rz);
    const float R11 = __fsub_rn(1.0f, __fadd_rn(xx_zz, xx_zz));
    const float R12 = __fadd_rn(yz_m_rx, yz_m_rx);
    const float R20 = __fadd_rn(xz_m_ry, xz_m_ry);
    const float R21 = __fadd_rn(yz_p_rx, yz_p_rx);
    const float R22 = __fsub_rn(1.0f, __fadd_rn(xx_yy, xx_yy));
    const float a0 = __fmul_rn(sx, R00), a1 = __fmul_rn(sy, R01), a2 = __fmul_rn(sz, R02);
    const float b0 = __fmul_rn(sx, R10), b1 = __fmul_rn(sy, R11), b2 = __fmul_rn(sz, R12);
    const float c0 = __fmul_rn(sx, R20), c1 = __fmul_rn(sy, R21), c2 = __fmul_rn(sz, R22);
    cov[0] = __fmaf_rn(a2, a2, __fmaf_rn(a0, a0, __fmul_rn(a1, a1)));
    cov[1] = __fmaf_rn(b2, a2, __fmaf_rn(b0, a0, __fmul_rn(b1, a1)));
    cov[2] = __fmaf_rn(c2, a2, __fmaf_rn(c0, a0, __fmul_rn(c1, a1)));
    cov[3] = __fmaf_rn(b2, b2, __fmaf_rn(b0, b0, __fmul_rn(b1, b1)));
    cov[4] = __fmaf_rn(c2, b2, __fmaf_rn(c0, b0, __fmul_rn(c1, b1)));
    cov[5] = __fmaf_rn(c2, c2, __fmaf_rn(c0, c0, __fmul_rn(c1, c1)));
}

// EWA projection (forward.cu:74-113): returns (a, b, c) of the 2-D covariance after +0.3.
// Also hands back the pieces the backward needs (T rows, clamp flags) when asked.
struct Cov2D {
    float a, b, c;
};
__device__ __forceinline__ Cov2D cov2d_project(float tx0, float ty0, float tz, float focal_x, float focal_y,
                                               float tan_fovx, float tan_fovy, const float *c3,
                                               const float *__restrict__ vm)
{
    const float limx = __fmul_rn(tan_fovx, 1.3f), limy = __fmul_rn(tan_fovy, 1.3f);
    const float txtz = __fdiv_rn(tx0, tz), tytz = __fdiv_rn(ty0, tz);
    const float cx = fminf(limx, fmaxf(-limx, txtz));
    const float cy = fminf(limy, fmaxf(-limy, tytz));
    const float tz2 = __fmul_rn(tz, tz);
    const float J00 = __fdiv_rn(focal_x, tz);
    const float J02 = __fdiv_rn(__fmul_rn(focal_x, __fmul_rn(cx, -tz)), tz2);
    const float J11 = __fdiv_rn(focal_y, tz);
    const float J12 = __fdiv_rn(__fmul_rn(focal_y, __fmul_rn(cy, -tz)), tz2);
    const float T00 = __fmaf_rn(vm[2], J02, __fmul_rn(vm[0], J00));
    const float T01 = __fmaf_rn(vm[6], J02, __fmul_rn(vm[4], J00));
    const float T02 = __fmaf_rn(J02, vm[10], __fmul_rn(vm[8], J00));
    const float T10 = __fmaf_rn(vm[2], J12, __fmul_rn(J11, vm[1]));
    const float T11 = __fmaf_rn(vm[6], J12, __fmul_rn(J11, vm[5]));
    const float T12 = __fmaf_rn(J12, vm[10], __fmul_rn(J11, vm[9]));
    const float u0 = __fmaf_rn(T02, c3[2], __fmaf_rn(T00, c3[0], __fmul_rn(T01, c3[1])));
    const float v0 = __fmaf_rn(T12, c3[2], __fmaf_rn(T10, c3[0], __fmul_rn(T11, c3[1])));
    const float u1 = __fmaf_rn(T02, c3[4], __fmaf_rn(T00, c3[1], __fmul_rn(T01, c3[3])));
    const float v1 = __fmaf_rn(T12, c3[4], __fmaf_rn(T10, c3[1], __fmul_rn(T11, c3[3])));
    const float u2 = __fmaf_rn(T02, c3[5], __fmaf_rn(T00, c3[2], __fmul_rn(T01, c3[4])));
    const float v2 = __fmaf_rn(T12, c3[5], __fmaf_rn(T10, c3[2], __fmul_rn(T11, c3[4])));
    Cov2D o;
    o.a = __fadd_rn(__fmaf_rn(T02, u2, __fmaf_rn(T00, u0, __fmul_rn(T01, u1))), 0.3f);
    o.b = __fmaf_rn(T02, v2, __fmaf_rn(T00, v0, __fmul_rn(T01, v1)));
    o.c = __fadd_rn(__fmaf_rn(T12, v2, __fmaf_rn(T10, v0, __fmul_rn(T11, v1))), 0.3f);
    return o;
}

// ((v + 1.0) * S - 1.0) * 0.5 with double intermediates (auxiliary.h:41-44)
__device__ __forceinline__ float ndc2pix(float v, int S)
{
    return (float)(__dmul_rn(__fma_rn((double)v + 1.0, (double)S, -1.0), 0.5));
}

// getRect (auxiliary.h:46-56) on a 16x16 tile grid
__device__ __forceinline__ void tile_rect(float px, float py, int radius, int gx, int gy, int &x0, int &y0, int &x1,
                                          int &y1)
{
    const float r = (float)radius;
    x0 = min(gx, max(0, (int)__fmul_rn(__fsub_rn(px, r), 0.0625f)));
    y0 = min(gy, max(0, (int)__fmul_rn(__fsub_rn(py, r), 0.0625f)));
    x1 = min(gx, max(0, (int)__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(px, r), 16.0f), -1.0f), 0.0625f)));
    y1 = min(gy, max(0, (int)__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(py, r), 16.0f), -1.0f), 0.0625f)));
}

// power = -0.5 (a dx^2 + c dy^2) - b dx dy, rounded as the reference's blend kernels round it
// (forward.cu:333-335 / backward.cu:486-488 compile to the same five operations).
__device__ __forceinline__ float splat_power(float dx, float dy, float a, float b, float c)
{
    const float q = __fmaf_rn(dx, __fmul_rn(dx, a), __fmul_rn(dy, __fmul_rn(dy, c)));
    return __fmaf_rn(q, -0.5f, -__fmul_rn(dy, __fmul_rn(dx, b)));
}


// ---------------------------------------------------------------------------------------------
// Footprint masks.  A 16x16 tile is cut into eight 8x4 pixel BLOCKS (= the warps of the blend
// kernels): block w = band * 2 + half, band = 4-row band 0..3, half = left / right 8 columns.
// A splat can only pass the alpha test at pixels with power >= tau, i.e. inside the ellipse
//   a u^2 + 2 b u v + c v^2 <= k,  k = -2 tau,  (u, v) = pixel - centre
// (tau already carries a 1e-4 margin on the power).  Bit w of a footprint mask is set when block w
// may hold such a pixel; a clear bit is a proof that it does not, so skipping the block never changes
// a result.  Mask 0 = the splat is dead in this tile (the reference's rectangle of 3 sigma_max is much
// larger than the ellipse for anisotropic or faint splats: a third of all instances on the headline scene).
//
// EllipseBands: per-Gaussian constants; band_columns() gives, for the image rows [ra, rb] (clipped
// to the ellipse's own row range), the absolute pixel-column interval [c_lo, c_hi] the ellipse reaches
// inside that band -- exact up to the stated slack: the rightmost point of the ellipse within the band
// sits at v = clamp(-(b/c) ex, band) because the boundary u_max(v) is concave.  The interval depends
// on the band only, not on the tile column, so a Gaussian computes it once per band of its rectangle.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float sqrt_fast(float x)  // MUFU.SQRT: 2^-22 relative, covered by the slack below
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

struct EllipseBands {
    float gx, gy;        // centre (pixels)
    float k_a, det_a2;   // k / a,  det / a^2
    float b_a;           // b / a
    float v_r;           // row offset of the rightmost point: -(b/c) ex   (the leftmost is at -v_r)
    int r_lo, r_hi;      // rows the ellipse reaches (may exceed the image)
    bool all;            // degenerate / non-finite: treat every block as reachable
    bool dead;           // never reaches alpha >= 1/255 anywhere
};

__device__ __forceinline__ EllipseBands ellipse_bands(float gx, float gy, float a, float b, float c, float tau)
{
    EllipseBands e;
    e.gx = gx;
    e.gy = gy;
    e.dead = tau > 0.0f;  // power <= 0 < tau for every pixel
    const float det = a * c - b * b, k = -2.0f * tau;
    e.all = !(det > 0.0f && a > 0.0f && c > 0.0f && k < 3.0e38f && k >= 0.0f);
    e.k_a = e.det_a2 = e.b_a = e.v_r = 0.f;
    e.r_lo = e.r_hi = 0;
    if (!e.all && !e.dead) {
        const float inv_det = __fdividef(1.0f, det), inv_a = __fdividef(1.0f, a);
        const float ex = sqrt_fast(k * c * inv_det) * 1.0001f + 0.02f;
        const float ey = sqrt_fast(k * a * inv_det) * 1.0001f + 0.02f;
        e.k_a = k * inv_a * 1.0002f;
        e.det_a2 = det * inv_a * inv_a;
        e.b_a = b * inv_a;
        e.v_r = -__fdividef(b, c) * ex;
        e.r_lo = (int)ceilf(fmaxf(gy - ey, -1.0e6f));
        e.r_hi = (int)floorf(fminf(gy + ey, 1.0e6f));
        e.all = !(ex < 1.0e6f && ey < 1.0e6f);
    }
    return e;
}

// columns reached inside rows [ra, rb] (ra <= rb, both inside [r_lo, r_hi]); empty when c_hi < c_lo
__device__ __forceinline__ void band_columns(const EllipseBands &e, int ra, int rb, int &c_lo, int &c_hi)
{
    const float v0 = (float)ra - e.gy, v1 = (float)rb - e.gy;
    const float vr = fminf(fmaxf(e.v_r, v0), v1), vl = fminf(fmaxf(-e.v_r, v0), v1);
    const float wr = sqrt_fast(fmaxf(e.k_a - e.det_a2 * vr * vr, 0.0f)) * 1.0001f + 0.02f;
    const float wl = sqrt_fast(fmaxf(e.k_a - e.det_a2 * vl * vl, 0.0f)) * 1.0001f + 0.02f;
    const float xmax = e.gx - e.b_a * vr + wr, xmin = e.gx - e.b_a * vl - wl;
    c_lo = (int)ceilf(fmaxf(xmin, -1.0e6f));
    c_hi = (int)floorf(fminf(xmax, 1.0e6f));
}

// footprint mask of one splat in the tile whose first pixel is (tile_x0, tile_y0): four bands, two halves
__device__ __forceinline__ uint32_t block_mask(const EllipseBands &e, int tile_x0, int tile_y0)
{
    if (e.dead) return 0u;
    if (e.all) return 0xffu;
    uint32_t m = 0;
#pragma unroll
    for (int band = 0; band < 4; band++) {
        const int ra = max(tile_y0 + 4 * band, e.r_lo), rb = min(tile_y0 + 4 * band + 3, e.r_hi);
        if (ra > rb) continue;
        int c_lo, c_hi;
        band_columns(e, ra, rb, c_lo, c_hi);
        if (c_hi < c_lo) continue;
        const uint32_t left = (c_lo <= tile_x0 + 7 && c_hi >= tile_x0) ? 1u : 0u;
        const uint32_t right = (c_lo <= tile_x0 + 15 && c_hi >= tile_x0 + 8) ? 2u : 0u;
        m |= (left | right) << (2 * band);
    }
    return m;
}

// Footprint mask straight from a staged splat record, for lists that carry none (P > 2^24 Gaussians;
// the blend kernels are instantiated once per list format so this costs the common one nothing).
__device__ __forceinline__ uint32_t block_mask_of_record(float x, float y, float a, float b, float c, float tau,
                                                         int tile_x0, int tile_y0)
{
    return block_mask(ellipse_bands(x, y, a, b, c, tau), tile_x0, tile_y0);
}

// Instance words carry the footprint mask next to the Gaussian id when the ids fit 24 bits:
//   low word of the sort key = id << 8 | mask   (the order by (depth, id) is unchanged: ids are unique)
// and the sorted list the blend kernels read holds the same low words.  For P >= 2^24 Gaussians the low
// word is the plain id and the blend kernels compute the mask while staging the record.  The format is a
// function of P alone, so the forward, the backward and sgr_inspect_state agree on it.
#define SGR_PACKED_MAX_P (1 << 24)
// strict: id 0xffffff with mask 0xff would read as the "no record" word
inline bool ids_packed(int P) { return P < SGR_PACKED_MAX_P; }

__device__ __forceinline__ float warp_sum(float v)
{
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// one 16-byte vector reduction into global memory (SASS REDG.E.ADD.F32x4)
__device__ __forceinline__ void red_add_v4(float *addr, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---- async-copy / mbarrier primitives (sm_90+ bulk copies: SASS UBLKCP; cp.async: LDGSTS) ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}
// 1-D bulk async copy global -> shared (TMA engine, no tensor map needed); bytes % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void cp_async16(void *dst_smem, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(void *dst_smem, const void *src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait()
{
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// 16-byte shared-memory load from a precomputed 32-bit shared-window address.  Indexing a
// __shared__ array with a runtime index inside the splat loop makes nvcc rebuild the window base
// (S2R SR_CgaCtaId + LEA ...) every iteration; the blend kernels compute the base once instead.
// Shared-window address of a __shared__ object, pinned in a register: the asm barrier stops nvcc
// from re-materialising the (S2R + LEA) sequence at every use inside the loops.
__device__ __forceinline__ uint32_t smem_addr_pinned(const void *p)
{
    uint32_t a = smem_u32(p), r;
    asm volatile("mov.u32 %0, %1;" : "=r"(r) : "r"(a));
    return r;
}
__device__ __forceinline__ float4 lds128(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr)
{
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}

__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v)
{
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
// Ampere-style async copies global -> shared by 32-bit shared-window address (SASS LDGSTS)
__device__ __forceinline__ void cp_async16_a(uint32_t dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8_a(uint32_t dst, const void *src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4_a(uint32_t dst, const void *src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void sts64(uint32_t addr, float a, float b)
{
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d)
{
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

#endif  // __CUDACC__

// The extra blended channel of sgr_rasterize_{forward,backward}_feature: one scalar per Gaussian, blended with the
// colour channels' alphas and transmittances over its own background.  A null pointer to it selects the plain blend.
struct FeatureChannel {
    const float *values;      // f32[P]
    const float *bg;          // device f32[1]
    float *out;               // forward: f32[H,W]
    const float *dL_dout;     // backward: f32[H,W]
    float *dL_dvalues;        // backward: f32[P]
};

// host-side stage entry points (defined in the .cu files)
int launch_forward(const SgrView *view, const SgrGaussians *g, SgrAlloc geom_alloc, void *geom_ctx,
                   SgrAlloc binning_alloc, void *binning_ctx, SgrAlloc image_alloc, void *image_ctx, float *out_color,
                   int32_t *radii, int64_t capacity_hint, int64_t *num_rendered, cudaStream_t stream,
                   const FeatureChannel *feat);
int launch_backward(const SgrView *view, const SgrGaussians *g, const int32_t *radii, const void *geom_buffer,
                    const void *binning_buffer, const void *image_buffer, int64_t num_rendered,
                    const float *dL_dout_color, float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity,
                    float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh, float *dL_dscales, float *dL_drotations,
                    void *grad_scratch, cudaStream_t stream, const SgrBackwardPlan *plan, const FeatureChannel *feat);

// The per-Gaussian backward pass: PB_T Gaussians per CTA, in backward_chunks() chunks of whole CTAs (at least one, at
// most one per CTA); chunk c covers the CTAs [b0, b1) (sgr_exchange.cu).
constexpr int PB_T = 64;
static inline int backward_chunks(int P, int num_chunks)
{
    const int n = num_chunks > 1 ? num_chunks : 1, blocks = (P + PB_T - 1) / PB_T;
    return n > blocks ? blocks : n;
}
void chunk_blocks(int blocks, int nchunks, int c, int taper, int *b0, int *b1);

// sgr_view_grad_finalize for the Gaussians [p0, p1) (sgr_exchange.cu); `who`: the message for bad arguments
int finalize_impl(int32_t P, int32_t p0, int32_t p1, int32_t M, int32_t sh_degree, int32_t num_views,
                  const float *means3D, const float *campos, const float *dRGB, int64_t view_stride, int32_t campos_stride,
                  float *dL_dsh, const float *reduced_records, float scale, float *dL_dmeans3D, float *dL_dopacity,
                  float *dL_dscales, float *dL_drotations, void *stream, const char *who);

// The peer exchange's share of one backward (sgr_peer.cu), called by launch_backward next to the stage hook; with
// plan == NULL nothing is enqueued.  rasterize_backward has checked the plan.
struct PeerBackward {
    const SgrPeerPlan *plan;
    cudaStream_t st;
    int P;
    float *dmeans3D, *dopacity, *dscales, *drots;  // where the split puts the reduced records
    int split_c = -1, split_p0 = 0, split_p1 = 0;  // the chunk whose split is still to be enqueued
    int blend_done(bool views);             // signal BLEND; views (MULTI): wait until every rank has
    int chunk_done(int c, int p0, int p1);  // signal CHUNK c; side stream: reduce chunk c, split chunk c - 1
    int finish();                           // side stream: split the last chunk
};

// The reference's full per-tile list (dead instances included) of a forward's state, into `full`; `cursor`: T words
int build_full_list(int P, int W, int H, const GeomState &geom, const ImageState &img, uint64_t num_rendered,
                    const BinState &full, uint32_t *cursor, cudaStream_t stream);

}  // namespace sgr
