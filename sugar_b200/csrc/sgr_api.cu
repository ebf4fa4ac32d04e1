// sgr_api.cu -- extern "C" entry points of libsugar_b200.so (declared in include/sugar_b200.h).
// Argument validation and error behaviour mirror the reference binding
// (diff-gaussian-rasterization/rasterize_points.cu:36-216): wrong shapes / ambiguous optionals
// are rejected up front, P == 0 returns without launching anything.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "sgr_internal.cuh"

namespace sgr {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what)
{
    set_error("[CUDA ERROR] %s: %s", what, cudaGetErrorString(e));
    return SGR_ECUDA;
}

int current_device(int *dev)
{
    SGR_CUDA(cudaGetDevice(dev));
    if (*dev < 0 || *dev >= SGR_MAX_DEVICES) {
        set_error("device ordinal %d out of range", *dev);
        return SGR_EINVAL;
    }
    return SGR_OK;
}

int once_per_device(DeviceOnce &once, int (*init)())
{
    static std::mutex mu;
    int dev = 0;
    int rc = current_device(&dev);
    if (rc) return rc;
    std::lock_guard<std::mutex> lock(mu);
    if (once.done[dev]) return SGR_OK;
    rc = init();
    once.done[dev] = rc == SGR_OK;
    return rc;
}

int device_sm_count()
{
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return 132;  // H100 SXM
    return n;
}

// ---- launch counter + optional event profiling (not thread-safe: one profiling client at a time)
static const char *const g_kind_names[K_NUM_KINDS] = {
    "preprocess", "tile_scan", "scatter", "tile_sort_smem", "tile_sort_global", "blend_forward", "blend_backward",
    "preprocess_backward", "field_pack", "field_forward", "field_backward", "field_unpack", "knn_build", "knn_query",
    "misc", "view_finalize", "peer_reduce", "peer_sync", "loss_forward", "loss_backward", "density_estimation_forward",
    "density_estimation_backward", "mesh_nc_forward", "mesh_nc_backward"};
struct ProfRec {
    cudaEvent_t a, b;
    int kind;
};
static unsigned long long g_launches = 0;
static bool g_prof_on = false;
static ProfRec *g_prof = nullptr;
static int g_prof_n = 0, g_prof_cap = 0;

void prof_begin(int kind, cudaStream_t st)
{
    g_launches++;
    if (!g_prof_on) return;
    if (g_prof_n == g_prof_cap) {
        const int ncap = g_prof_cap ? g_prof_cap * 2 : 1024;
        ProfRec *np = (ProfRec *)realloc(g_prof, sizeof(ProfRec) * ncap);
        if (!np) return;
        for (int i = g_prof_cap; i < ncap; i++) {
            cudaEventCreate(&np[i].a);
            cudaEventCreate(&np[i].b);
        }
        g_prof = np;
        g_prof_cap = ncap;
    }
    g_prof[g_prof_n].kind = kind;
    cudaEventRecord(g_prof[g_prof_n].a, st);
}

void note_launches(int extra) { g_launches += (unsigned long long)extra; }

void prof_end(cudaStream_t st)
{
    if (!g_prof_on || g_prof_n >= g_prof_cap) return;
    cudaEventRecord(g_prof[g_prof_n].b, st);
    g_prof_n++;
}

// the 16-bit tile rect bounds the image at 65535 tiles per side
static bool image_size_ok(int W, int H) { return W > 0 && H > 0 && W <= 65535 * 16 && H <= 65535 * 16; }

static int validate(const SgrView *view, const SgrGaussians *g, bool forward)
{
    if (!view || !g) {
        set_error("null view/gaussians");
        return SGR_EINVAL;
    }
    if (g->P < 0 || view->image_width <= 0 || view->image_height <= 0) {
        set_error("bad sizes P=%d W=%d H=%d", g->P, view->image_width, view->image_height);
        return SGR_EINVAL;
    }
    if (!image_size_ok(view->image_width, view->image_height)) {
        set_error("image too large for the 16-bit tile rect");
        return SGR_EINVAL;
    }
    if (g->P == 0) return SGR_OK;
    if (!g->means3D || (forward && !g->opacities) || !view->bg || !view->viewmatrix || !view->projmatrix || !view->campos) {
        set_error("means3D / opacities / bg / viewmatrix / projmatrix / campos must be non-null");
        return SGR_EINVAL;
    }
    if ((g->shs == nullptr) == (g->colors_precomp == nullptr)) {
        set_error("Please provide excatly one of either SHs or precomputed colors!");
        return SGR_EINVAL;
    }
    const bool sr = g->scales && g->rotations;
    if (((g->scales != nullptr) != (g->rotations != nullptr)) || (sr == (g->cov3D_precomp != nullptr))) {
        set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
        return SGR_EINVAL;
    }
    if (g->shs && (g->M <= 0 || (view->sh_degree + 1) * (view->sh_degree + 1) > g->M || view->sh_degree < 0 ||
                   view->sh_degree > 3)) {
        set_error("sh_degree %d needs %d coefficients but M=%d", view->sh_degree,
                  (view->sh_degree + 1) * (view->sh_degree + 1), g->M);
        return SGR_EINVAL;
    }
    return SGR_OK;
}

// The plain and the feature forward (feat != NULL): argument checks, then P == 0 fills the outputs without launching
// anything (rasterize_points.cu:81).  The feature adds only its own pointers and its rejection of raw-parameter mode.
static int rasterize_forward(const char *who, const SgrView *view, const SgrGaussians *g, SgrAlloc geom_alloc,
                             void *geom_ctx, SgrAlloc binning_alloc, void *binning_ctx, SgrAlloc image_alloc,
                             void *image_ctx, float *out_color, int32_t *radii, int64_t capacity_hint,
                             int64_t *num_rendered, void *stream, const FeatureChannel *feat)
{
    int rc = validate(view, g, true);
    if (rc) return rc;
    if (!out_color || !num_rendered || !geom_alloc || !binning_alloc || !image_alloc || (feat && !feat->out)) {
        set_error("null output / allocator");
        return SGR_EINVAL;
    }
    if (feat && g->activations != 0) {
        set_error("%s: raw-parameter mode is not supported", who);
        return SGR_EINVAL;
    }
    *num_rendered = 0;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t npix = (size_t)view->image_width * view->image_height;
    if (g->P == 0) {
        SGR_CUDA(cudaMemsetAsync(out_color, 0, sizeof(float) * 3 * npix, st));
        if (feat) SGR_CUDA(cudaMemsetAsync(feat->out, 0, sizeof(float) * npix, st));
        return SGR_OK;
    }
    if (!radii || (feat && (!feat->values || !feat->bg))) {
        set_error(feat ? "radii / values / feature_bg must be non-null" : "radii must be non-null");
        return SGR_EINVAL;
    }
    return launch_forward(view, g, geom_alloc, geom_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, out_color,
                          radii, capacity_hint, num_rendered, st, feat);
}

// The plain / staged and the feature backward (feat != NULL): argument checks, P == 0 launches nothing.  The feature
// adds only its own pointers and its rejection of raw-parameter mode.
static int rasterize_backward(const char *who, const SgrView *view, const SgrGaussians *g, const int32_t *radii,
                              const void *geom_buffer, const void *binning_buffer, const void *image_buffer,
                              int64_t num_rendered, const float *dL_dout_color, float *dL_dmeans2D, float *dL_dcolors,
                              float *dL_dopacity, float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh,
                              float *dL_dscales, float *dL_drotations, void *grad_scratch, void *stream,
                              const SgrBackwardPlan *plan, const FeatureChannel *feat)
{
    int rc = validate(view, g, false);
    if (rc) return rc;
    if (feat && g->activations != 0) {
        set_error("%s: raw-parameter mode is not supported", who);
        return SGR_EINVAL;
    }
    if (g->P == 0) return SGR_OK;
    const bool records = plan && plan->reduce_records;
    if (!radii || !geom_buffer || !binning_buffer || !image_buffer || !dL_dout_color || !dL_dmeans2D || !dL_dcolors ||
        !dL_dcov3D || !grad_scratch || (!records && (!dL_dopacity || !dL_dmeans3D || !dL_dscales || !dL_drotations)) ||
        (feat && (!feat->values || !feat->bg || !feat->dL_dout || !feat->dL_dvalues))) {
        set_error("null pointer passed to %s", who);
        return SGR_EINVAL;
    }
    // the plan as well, before anything is enqueued: a peer-mode backward that gave up after its BLEND signal had gone
    // out would leave the other ranks waiting for it until their wait kernels trap
    if (g->activations != 0 && g->shs && dL_dsh && g->M > 1 && !(plan && plan->dL_dsh_rest)) {
        set_error("raw-parameter mode needs SgrBackwardPlan.dL_dsh_rest");
        return SGR_EINVAL;
    }
    const SgrPeerPlan *pp = plan ? plan->peer : nullptr;
    const int nchunks = backward_chunks(g->P, plan ? plan->num_chunks : 1);
    const auto slots_ok = [&](int slot0, int nslots) { return slot0 >= 0 && slot0 + nslots <= SGR_PEER_MAX_SLOTS; };
    if (pp && (!pp->peer_flag_tab || pp->peer_nranks < 1 || pp->peer_nranks > SGR_PEER_MAX_RANKS || pp->peer_rank < 0 ||
               pp->peer_rank >= pp->peer_nranks || !slots_ok(pp->peer_slot_blend, 1) ||
               !slots_ok(pp->peer_slot_chunk0, nchunks) || (pp->peer_signal_stream && nchunks > 19))) {
        set_error("SgrPeerPlan: needs peer_flag_tab, 1 <= peer_nranks <= %d, peer_rank < peer_nranks, flag slots in the "
                  "table and, with peer_signal_stream, at most 19 chunks", SGR_PEER_MAX_RANKS);
        return SGR_EINVAL;
    }
    const bool views = pp && pp->peer_view_blocks && dL_dsh && g->shs;
    if (views && (g->activations != 0 || !pp->peer_flags)) {
        set_error("peer_view_blocks: needs peer_flags and activated (not raw) parameters");
        return SGR_EINVAL;
    }
    if (views && pp->peer_record_stages && !records) {
        set_error("peer_record_stages needs reduce_records (the local staging array)");
        return SGR_EINVAL;
    }
    if (pp && pp->peer_side_stream &&
        (!pp->peer_rec_tab || !pp->peer_sum_tab || !pp->peer_sums || !pp->peer_flags || !records || !dL_dmeans3D ||
         !dL_dopacity || !dL_dscales || !dL_drotations || nchunks > 16 || !slots_ok(pp->peer_slot_reduced0, nchunks))) {
        set_error("peer_side_stream needs peer_rec_tab / peer_sum_tab / peer_sums / peer_flags, reduce_records, the four "
                  "record-bound gradient arrays, at most 16 chunks and peer_slot_reduced0 + chunks inside the flag table");
        return SGR_EINVAL;
    }
    return launch_backward(view, g, radii, geom_buffer, binning_buffer, image_buffer, num_rendered, dL_dout_color,
                           dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales,
                           dL_drotations, grad_scratch, (cudaStream_t)stream, plan, feat);
}

__global__ void fill_background_kernel(int W, int H, const float *__restrict__ bg, float *__restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)W * H;
    if (i < n) {
        out[i] = bg[0];
        out[n + i] = bg[1];
        out[2 * n + i] = bg[2];
    }
}

__global__ void inspect_geom_kernel(int P, GeomState g, const int32_t *radii_unused, float *depths, float *means2D,
                                    float *conic_opacity, float *rgb, uint8_t *clamped, uint32_t *tiles_touched)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const ushort4 rc = g.rect[i];
    const uint32_t nt = (uint32_t)(rc.z - rc.x) * (uint32_t)(rc.w - rc.y);
    if (tiles_touched) tiles_touched[i] = nt;
    const bool vis = nt != 0;
    float4 r0 = make_float4(0, 0, 0, 0), r1 = r0, r2 = r0;
    float d = 0.f;
    uint32_t aux = 0;
    if (vis) {
        r0 = g.rec[(size_t)i * 3];
        r1 = g.rec[(size_t)i * 3 + 1];
        r2 = g.rec[(size_t)i * 3 + 2];
        d = g.depth[i];
        aux = __float_as_uint(r2.z);
    }
    if (depths) depths[i] = d;
    if (means2D) {
        means2D[2 * i] = r0.x;
        means2D[2 * i + 1] = r0.y;
    }
    if (conic_opacity) {
        conic_opacity[4 * i] = r0.z;
        conic_opacity[4 * i + 1] = r0.w;
        conic_opacity[4 * i + 2] = r1.x;
        conic_opacity[4 * i + 3] = r1.z;
    }
    if (rgb) {
        rgb[3 * i] = r1.w;
        rgb[3 * i + 1] = r2.x;
        rgb[3 * i + 2] = r2.y;
    }
    if (clamped) {
        clamped[3 * i] = aux & 1u;
        clamped[3 * i + 1] = (aux >> 1) & 1u;
        clamped[3 * i + 2] = (aux >> 2) & 1u;
    }
}

__global__ void inspect_bin_kernel(int T, int packed, const uint32_t *__restrict__ tile_start,
                                   const uint32_t *__restrict__ plist, const float *__restrict__ depth, uint64_t *keys,
                                   uint32_t *point_list, uint32_t *ranges, uint8_t *footprint)
{
    const int t = blockIdx.x;
    const uint32_t lo = tile_start[t], hi = tile_start[t + 1];
    if (ranges && threadIdx.x == 0) {
        // identifyTileRanges leaves empty tiles at (0,0) (rasterizer_impl.cu:310)
        ranges[2 * t] = hi > lo ? lo : 0u;
        ranges[2 * t + 1] = hi > lo ? hi : 0u;
    }
    for (uint32_t k = lo + threadIdx.x; k < hi; k += blockDim.x) {
        const uint32_t w = plist[k], id = packed ? (w >> 8) : w;
        if (point_list) point_list[k] = id;
        if (footprint) footprint[k] = packed ? (uint8_t)(w & 0xffu) : (uint8_t)0xffu;
        if (keys) keys[k] = ((uint64_t)t << 32) | __float_as_uint(depth[id]);
    }
}

// n_contrib of the blend kernels counts positions in the tile's LIVE list (dead instances left out); the reference
// counts the entries of the full list up to its last contributor.  The last contributor is the same instance in both,
// so its position in the full sorted segment -- found by (depth bits, id), the sort key -- plus one is the reference's.
__global__ void inspect_n_contrib_kernel(int W, int H, int gx, int packed, const uint32_t *__restrict__ tile_start,
                                         const uint32_t *__restrict__ live, const uint32_t *__restrict__ full,
                                         const float *__restrict__ depth, const uint32_t *__restrict__ n_live,
                                         uint32_t *__restrict__ n_ref)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W * H) return;
    const uint32_t n = n_live[i];
    uint32_t out = 0;
    if (n) {
        const int x = i % W, y = i / W, t = (y / SGR_TILE) * gx + x / SGR_TILE;
        const uint32_t lo = tile_start[t], hi = tile_start[t + 1];
        const auto key = [&](uint32_t w) {
            const uint32_t id = packed ? (w >> 8) : w;
            return ((uint64_t)__float_as_uint(depth[id]) << 32) | id;
        };
        const uint64_t k = key(live[lo + n - 1]);
        uint32_t a = lo, b = hi;  // first position of [lo, hi) whose key is not below k
        while (a < b) {
            const uint32_t m = (a + b) >> 1;
            if (key(full[m]) < k) a = m + 1;
            else b = m;
        }
        out = a - lo + 1;
    }
    n_ref[i] = out;
}

__global__ void mark_visible_kernel(int P, const float *__restrict__ means, const float *__restrict__ vm,
                                    uint8_t *__restrict__ present);  // sgr_forward.cu

#ifdef SGR_BLEND_STATS
int read_fwd_stats(unsigned long long *out, int reset);  // sgr_forward.cu
int read_bwd_stats(unsigned long long *out, int reset);  // sgr_backward.cu
#endif

}  // namespace sgr

using namespace sgr;

extern "C" {

const char *sgr_last_error(void) { return g_err; }

unsigned long long sgr_launch_count(void) { return g_launches; }
int sgr_num_kernel_kinds(void) { return K_NUM_KINDS; }

// sizes of the ABI structs as this library was compiled: a binding checks its own layout against them
size_t sgr_struct_bytes(int32_t which)
{
    switch (which) {
        case 0: return sizeof(SgrView);
        case 1: return sizeof(SgrGaussians);
        case 2: return sizeof(SgrBackwardPlan);
        case 3: return sizeof(SgrFieldParams);
        case 4: return sizeof(SgrSsimParams);
        case 5: return sizeof(SgrDensifyGates);
        case 6: return sizeof(SgrDensifyColumn);
        case 7: return sizeof(SgrAdamSegment);
        case 8: return sizeof(SgrPeerPlan);
        default: return 0;
    }
}
const char *sgr_kernel_name(int kind) { return (kind >= 0 && kind < K_NUM_KINDS) ? g_kind_names[kind] : "?"; }

int sgr_profile_enable(int on)
{
    if (on && g_prof_cap == 0) {  // create the event pool up front, outside any timed region
        const int ncap = 8192;
        ProfRec *np = (ProfRec *)malloc(sizeof(ProfRec) * ncap);
        if (!np) {
            set_error("out of host memory for the profile log");
            return SGR_ENOMEM;
        }
        for (int i = 0; i < ncap; i++) {
            SGR_CUDA(cudaEventCreate(&np[i].a));
            SGR_CUDA(cudaEventCreate(&np[i].b));
        }
        g_prof = np;
        g_prof_cap = ncap;
    }
    g_prof_on = on != 0;
    if (on) g_prof_n = 0;
    return SGR_OK;
}

int sgr_profile_timeline(int max_records, int *kinds, float *t_begin_ms, float *t_end_ms)
{
    // per-launch begin/end times relative to the first recorded launch (does not reset the log)
    const int n = g_prof_n < max_records ? g_prof_n : max_records;
    for (int i = 0; i < n; i++) {
        SGR_CUDA(cudaEventSynchronize(g_prof[i].b));
        kinds[i] = g_prof[i].kind;
        SGR_CUDA(cudaEventElapsedTime(&t_begin_ms[i], g_prof[0].a, g_prof[i].a));
        SGR_CUDA(cudaEventElapsedTime(&t_end_ms[i], g_prof[0].a, g_prof[i].b));
    }
    return n;
}

int sgr_profile_read(float *total_ms, int *counts)
{
    for (int k = 0; k < K_NUM_KINDS; k++) {
        total_ms[k] = 0.f;
        counts[k] = 0;
    }
    for (int i = 0; i < g_prof_n; i++) {
        SGR_CUDA(cudaEventSynchronize(g_prof[i].b));
        float ms = 0.f;
        SGR_CUDA(cudaEventElapsedTime(&ms, g_prof[i].a, g_prof[i].b));
        total_ms[g_prof[i].kind] += ms;
        counts[g_prof[i].kind]++;
    }
    g_prof_n = 0;
    return SGR_OK;
}
#ifdef SGR_BLEND_STATS
SGR_API int sgr_debug_blend_stats(unsigned long long *out16, int reset)
{
    int rc = sgr::read_fwd_stats(out16, reset);
    if (rc) return rc;
    return sgr::read_bwd_stats(out16 + 8, reset);
}
#endif
const char *sgr_version(void) { return "sugar_b200 0.1 (sm_90a)"; }

size_t sgr_geometry_bytes(int32_t P) { return P < 0 ? 0 : layout_bytes([&](Layout &l) { GeomState::carve(l, P); }); }
size_t sgr_binning_bytes(int64_t C) { return C < 0 ? 0 : layout_bytes([&](Layout &l) { BinState::carve(l, C); }); }
size_t sgr_image_bytes(int32_t W, int32_t H)
{
    return image_size_ok(W, H) ? layout_bytes([&](Layout &l) { ImageState::carve(l, W, H); }) : 0;
}
size_t sgr_backward_scratch_bytes(int32_t P) { return P < 0 ? 0 : layout_bytes([&](Layout &l) { carve_grad_acc(l, P); }); }

int sgr_rasterize_forward(const SgrView *view, const SgrGaussians *g, SgrAlloc geom_alloc, void *geom_ctx,
                          SgrAlloc binning_alloc, void *binning_ctx, SgrAlloc image_alloc, void *image_ctx,
                          float *out_color, int32_t *radii, int64_t capacity_hint, int64_t *num_rendered, void *stream)
{
    return rasterize_forward("sgr_rasterize_forward", view, g, geom_alloc, geom_ctx, binning_alloc, binning_ctx,
                             image_alloc, image_ctx, out_color, radii, capacity_hint, num_rendered, stream, nullptr);
}

int sgr_rasterize_forward_feature(const SgrView *view, const SgrGaussians *g, SgrAlloc geom_alloc, void *geom_ctx,
                                  SgrAlloc binning_alloc, void *binning_ctx, SgrAlloc image_alloc, void *image_ctx,
                                  const float *values, const float *feature_bg, float *out_color, float *out_feature,
                                  int32_t *radii, int64_t capacity_hint, int64_t *num_rendered, void *stream)
{
    const FeatureChannel feat = {values, feature_bg, out_feature, nullptr, nullptr};
    return rasterize_forward("sgr_rasterize_forward_feature", view, g, geom_alloc, geom_ctx, binning_alloc, binning_ctx,
                             image_alloc, image_ctx, out_color, radii, capacity_hint, num_rendered, stream, &feat);
}

int sgr_rasterize_backward_staged(const SgrView *view, const SgrGaussians *g, const int32_t *radii, const void *geom_buffer,
                           const void *binning_buffer, const void *image_buffer, int64_t num_rendered,
                           const float *dL_dout_color, float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity,
                           float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh, float *dL_dscales,
                           float *dL_drotations, void *grad_scratch, void *stream, const SgrBackwardPlan *plan)
{
    return rasterize_backward("sgr_rasterize_backward", view, g, radii, geom_buffer, binning_buffer, image_buffer,
                              num_rendered, dL_dout_color, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D,
                              dL_dsh, dL_dscales, dL_drotations, grad_scratch, stream, plan, nullptr);
}

int sgr_rasterize_backward_feature(const SgrView *view, const SgrGaussians *g, const int32_t *radii,
                                   const void *geom_buffer, const void *binning_buffer, const void *image_buffer,
                                   int64_t num_rendered, const float *dL_dout_color, const float *values,
                                   const float *feature_bg, const float *dL_dout_feature, float *dL_dmeans2D,
                                   float *dL_dcolors, float *dL_dopacity, float *dL_dmeans3D, float *dL_dcov3D,
                                   float *dL_dsh, float *dL_dscales, float *dL_drotations, float *dL_dvalues,
                                   void *grad_scratch, void *stream)
{
    const FeatureChannel feat = {values, feature_bg, nullptr, dL_dout_feature, dL_dvalues};
    return rasterize_backward("sgr_rasterize_backward_feature", view, g, radii, geom_buffer, binning_buffer,
                              image_buffer, num_rendered, dL_dout_color, dL_dmeans2D, dL_dcolors, dL_dopacity,
                              dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations, grad_scratch, stream, nullptr,
                              &feat);
}

int sgr_rasterize_backward(const SgrView *view, const SgrGaussians *g, const int32_t *radii, const void *geom_buffer,
                           const void *binning_buffer, const void *image_buffer, int64_t num_rendered,
                           const float *dL_dout_color, float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity,
                           float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh, float *dL_dscales,
                           float *dL_drotations, void *grad_scratch, void *stream)
{
    return sgr_rasterize_backward_staged(view, g, radii, geom_buffer, binning_buffer, image_buffer, num_rendered,
                                         dL_dout_color, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D,
                                         dL_dsh, dL_dscales, dL_drotations, grad_scratch, stream, nullptr);
}

int sgr_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix,
                     uint8_t *present, void *stream)
{
    (void)projmatrix;
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) {
        set_error("bad arguments to sgr_mark_visible");
        return SGR_EINVAL;
    }
    if (P == 0) return SGR_OK;
    SGR_LAUNCH(K_MISC, (cudaStream_t)stream,
               sgr::mark_visible_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, means3D, viewmatrix, present));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_inspect_state(int32_t P, int32_t width, int32_t height, int64_t num_rendered, const void *geom_buffer,
                      const void *binning_buffer, const void *image_buffer, float *depths, float *means2D,
                      float *conic_opacity, float *rgb, uint8_t *clamped, uint32_t *tiles_touched, uint64_t *keys,
                      uint32_t *point_list, uint32_t *ranges, float *final_T, uint32_t *n_contrib, uint8_t *footprint,
                      void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0 || !geom_buffer || !image_buffer) {
        set_error("bad arguments to sgr_inspect_state");
        return SGR_EINVAL;
    }
    Layout geom_l(geom_buffer), img_l(image_buffer);
    GeomState geom = GeomState::carve(geom_l, P);
    ImageState img = ImageState::carve(img_l, width, height);
    const int T = ((width + 15) / 16) * ((height + 15) / 16);
    inspect_geom_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, geom, nullptr, depths, means2D, conic_opacity, rgb, clamped,
                                                         tiles_touched);
    const size_t npix = (size_t)width * height;
    if (final_T) SGR_CUDA(cudaMemcpyAsync(final_T, img.final_T, npix * 4, cudaMemcpyDeviceToDevice, st));
    if (num_rendered == 0) {
        if (n_contrib) SGR_CUDA(cudaMemsetAsync(n_contrib, 0, npix * 4, st));
        SGR_CUDA(cudaGetLastError());
        return SGR_OK;
    }
    if (!(keys || point_list || ranges || footprint || n_contrib)) {
        SGR_CUDA(cudaGetLastError());
        return SGR_OK;
    }
    if (!binning_buffer) {
        set_error("sgr_inspect_state: the list and n_contrib need the binning buffer");
        return SGR_EINVAL;
    }
    // The forward kept only the live instances; the reference's list (dead ones included, with their masks) is
    // rebuilt here in scratch of its own by the forward's scatter and sorts.  A diagnostic path: it allocates.
    const int gx = (width + 15) / 16;
    const size_t R = (size_t)num_rendered;
    uint32_t *cursor = nullptr;  // the tile cursors, then a binning layout
    const auto full_list = [&](Layout &l) { return cursor = l.take<uint32_t>(T), BinState::carve(l, R); };
    void *mem = nullptr;
    SGR_CUDA(cudaMallocAsync(&mem, layout_bytes(full_list), st));
    Layout mem_l(mem), live_l(binning_buffer);
    const BinState full = full_list(mem_l);
    const BinState live = BinState::carve(live_l, R);
    const int packed = ids_packed(P) ? 1 : 0;
    int rc = build_full_list(P, width, height, geom, img, R, full, cursor, st);
    if (rc == SGR_OK) {
        if (keys || point_list || ranges || footprint)
            inspect_bin_kernel<<<T, 128, 0, st>>>(T, packed, img.tile_start, full.plist, geom.depth, keys, point_list,
                                                  ranges, footprint);
        if (n_contrib)
            inspect_n_contrib_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(
                width, height, gx, packed, img.tile_start, live.plist, full.plist, geom.depth, img.n_contrib, n_contrib);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) rc = cuda_fail(e, "sgr_inspect_state");
    }
    const cudaError_t ef = cudaFreeAsync(mem, st);
    if (rc) return rc;
    SGR_CUDA(ef);
    return SGR_OK;
}

}  // extern "C"
