/*
 * sugar_b200.h -- C ABI of libsugar_b200.so: a Hopper (sm_90a) differentiable
 * Gaussian-splat rasterizer + SuGaR density/SDF field evaluator.
 *
 * Drop-in boundary.  These entry points are what a binding of the reference's rasterizer
 * path would call instead of `CudaRasterizer::Rasterizer::{forward,backward,markVisible}`
 * (gaussian_splatting/submodules/diff-gaussian-rasterization/cuda_rasterizer/rasterizer.h:20-85),
 * and instead of the PyTorch ops behind `SuGaR.get_field_values` / `SuGaR.compute_density`
 * (sugar_scene/sugar_model.py:1247-1316, 1345-1368).  Plain pointers and sizes only: every
 * pointer is a DEVICE pointer unless stated otherwise; the library allocates nothing that
 * outlives a call except one pinned 4 KiB page + one event per device (the num_rendered
 * read-back).  All work is enqueued on the caller's `stream` (a cudaStream_t passed as void*).
 *
 * Every function returns 0 on success or a negative SGR_E* code; sgr_last_error() gives the
 * thread-local message.  CUDA launch errors surface synchronously only when `debug` is set
 * (reference: CHECK_CUDA, cuda_rasterizer/auxiliary.h:166-173).
 */
#ifndef SUGAR_B200_H_
#define SUGAR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SGR_API __attribute__((visibility("default")))
#else
#define SGR_API
#endif

#define SGR_OK 0
#define SGR_EINVAL (-1)   /* bad argument (shape, null pointer, ambiguous optionals) */
#define SGR_ECUDA (-2)    /* CUDA runtime error */
#define SGR_ENOMEM (-3)   /* an allocator callback returned NULL */

/* Per-view constants: field-for-field `GaussianRasterizationSettings`
 * (diff_gaussian_rasterization/__init__.py:157-169). */
typedef struct SgrView {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    const float *bg;         /* f32[3] */
    float scale_modifier;
    const float *viewmatrix; /* f32[16], world->view transposed (read column-major) */
    const float *projmatrix; /* f32[16], full projection transposed */
    int32_t sh_degree;       /* active degree D, 0..3 */
    const float *campos;     /* f32[3] */
    int32_t prefiltered;
    int32_t debug;
} SgrView;

/* Per-Gaussian inputs of `_C.rasterize_gaussians` (rasterize_points.h:19-38).  Optional
 * arrays are NULL when absent, exactly as the reference tests `ptr == nullptr`
 * (forward.cu:205,241): exactly one of {shs, colors_precomp} and exactly one of
 * {scales+rotations, cov3D_precomp} must be non-NULL. */
typedef struct SgrGaussians {
    int32_t P;                   /* number of Gaussians */
    int32_t M;                   /* SH coefficients stored per Gaussian (0 if shs == NULL) */
    const float *means3D;        /* f32[P,3] */
    const float *opacities;      /* f32[P]   */
    const float *shs;            /* f32[P,M,3] or NULL */
    const float *colors_precomp; /* f32[P,3]   or NULL */
    const float *scales;         /* f32[P,3]   or NULL */
    const float *rotations;      /* f32[P,4] (w,x,y,z; pre-normalised by the caller) or NULL */
    const float *cov3D_precomp;  /* f32[P,6]   or NULL */
    /* Raw-parameter mode (0 = the reference's contract above).  SGR_ACT_RAW: the arrays are a SuGaR model's raw
     * parameters and its activations (sugar_scene/sugar_model.py:400-479) are applied in the kernels, their chain
     * rule in the backward: opacities = all_densities (sigmoid), scales = _scales (exp), rotations = _quaternions
     * (normalize), and the SH coefficients stay in the model's two arrays: shs = _sh_coordinates_dc f32[P,1,3],
     * sh_rest = _sh_coordinates_rest f32[P,M-1,3].  The backward's dL_dopacity / dL_dscales / dL_drotations are
     * then gradients of the RAW parameters, dL_dsh is f32[P,1,3] and dL_dsh_rest (SgrBackwardPlan) f32[P,M-1,3]. */
    int32_t activations;
    const float *sh_rest;        /* f32[P,M-1,3], raw mode only */
} SgrGaussians;
#define SGR_ACT_RAW 1

/* Scratch allocator: replaces `std::function<char*(size_t)>` (rasterizer.h:31-34,
 * rasterize_points.cu:27-33).  Must return device memory aligned to >= 256 bytes that stays
 * valid until the matching backward has run.  The three buffers are opaque round-trip state. */
typedef void *(*SgrAlloc)(void *ctx, size_t bytes);

/* Forward: replaces Rasterizer::forward (rasterizer_impl.cu:198-336).
 *   out_color  f32[3,H,W]  (fully written)
 *   radii      i32[P]      (fully written; >0 == visible)
 *   capacity_hint: 0 -> wait for the instance count before sizing the binning buffer (what the
 *     reference does, rasterizer_impl.cu:281); >0 -> allocate that many instances up front and
 *     enqueue everything without a host wait, re-running binning+blend only on overflow.
 *   *num_rendered receives R (number of (Gaussian, tile) instances). */
SGR_API int sgr_rasterize_forward(const SgrView *view, const SgrGaussians *g,
                          SgrAlloc geom_alloc, void *geom_ctx,
                          SgrAlloc binning_alloc, void *binning_ctx,
                          SgrAlloc image_alloc, void *image_ctx,
                          float *out_color, int32_t *radii,
                          int64_t capacity_hint, int64_t *num_rendered, void *stream);

/* Backward: replaces Rasterizer::backward (rasterizer_impl.cu:340-434) together with the
 * zero-initialised outputs of RasterizeGaussiansBackwardCUDA (rasterize_points.cu:151-159):
 * every output row is written by the kernels (zeros for culled Gaussians), so the caller may
 * pass uninitialised memory.  `grad_scratch` must hold sgr_backward_scratch_bytes(P).
 *   dL_dmeans2D f32[P,3], dL_dcolors f32[P,3], dL_dopacity f32[P,1], dL_dmeans3D f32[P,3],
 *   dL_dcov3D f32[P,6], dL_dsh f32[P,M,3], dL_dscales f32[P,3], dL_drotations f32[P,4].
 * dL_dcolors is the gradient of colors_precomp when colours were precomputed; with SH colours it is the
 * clamp-masked dL/dRGB per Gaussian (the reference's value is unmasked there, but no caller can observe
 * it: colors_precomp is absent).  dL_dsh may be NULL: when M == 0, or with SH present to select "factor
 * mode" -- dL_dsh is not produced, and sgr_view_grad_finalize rebuilds (the sum over views of) dL_dsh
 * from dL_dcolors.  All other outputs are unchanged.  Output pointers that are 16-byte aligned
 * leave through TMA bulk stores. */
SGR_API int sgr_rasterize_backward(const SgrView *view, const SgrGaussians *g, const int32_t *radii,
                           const void *geom_buffer, const void *binning_buffer, const void *image_buffer,
                           int64_t num_rendered, const float *dL_dout_color,
                           float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity,
                           float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh,
                           float *dL_dscales, float *dL_drotations,
                           void *grad_scratch, void *stream);

/* Forward and backward with one extra blended channel: a scalar per Gaussian (e.g. its view-space depth) blended
 * with the same alphas and transmittances as the colours, over its own background.  One call renders what two
 * sgr_rasterize_forward calls would (the second with colors_precomp = values in every channel and bg = *feature_bg),
 * and out_color / out_feature are bit-identical to theirs (out_feature to channel 0 of the second).
 *   values      f32[P]      the blended scalar (an input: its gradient is dL_dvalues)
 *   feature_bg  f32[1]      DEVICE pointer to the channel's background
 *   out_feature f32[H,W]    (fully written; zeros when P == 0, like out_color)
 * The backward equals the sum of the two calls' backwards up to fp32 summation order:
 *   dL_dout_feature f32[H,W] in, dL_dvalues f32[P] out (every row written, zeros for culled Gaussians);
 *   the other outputs as in sgr_rasterize_backward, dL_dmeans2D / dL_dopacity / dL_dmeans3D ... holding both
 *   channels' terms.
 * Raw-parameter mode (SgrGaussians.activations != 0) is not supported. */
SGR_API int sgr_rasterize_forward_feature(const SgrView *view, const SgrGaussians *g,
                          SgrAlloc geom_alloc, void *geom_ctx,
                          SgrAlloc binning_alloc, void *binning_ctx,
                          SgrAlloc image_alloc, void *image_ctx,
                          const float *values, const float *feature_bg,
                          float *out_color, float *out_feature, int32_t *radii,
                          int64_t capacity_hint, int64_t *num_rendered, void *stream);
SGR_API int sgr_rasterize_backward_feature(const SgrView *view, const SgrGaussians *g, const int32_t *radii,
                           const void *geom_buffer, const void *binning_buffer, const void *image_buffer,
                           int64_t num_rendered, const float *dL_dout_color,
                           const float *values, const float *feature_bg, const float *dL_dout_feature,
                           float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity,
                           float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh,
                           float *dL_dscales, float *dL_drotations, float *dL_dvalues,
                           void *grad_scratch, void *stream);

/* The same backward with a plan: stage hooks, a chunked per-Gaussian pass and record-form outputs.  This is
 * what the view-parallel (one view per GPU) step drives, sugar_b200/parallel.py; the reference has no
 * counterpart (it renders one view on one GPU, sugar_trainers/coarse_sdf.py:98,507).
 *
 * hook(hook_ctx, stage) is called on the HOST, between kernel enqueues on `stream`:
 *   SGR_STAGE_BLEND_DONE        the blend pass is enqueued: everything on `stream` so far makes dL_dcolors final.
 *                               With SH colours dL_dcolors holds the clamp-masked dL/dRGB per Gaussian -- this
 *                               view's rank-1 SH factor: a caller that exchanges factors instead of dL_dsh
 *                               (dL_dsh == NULL, "factor mode") starts its all-gather here, underneath the
 *                               per-Gaussian pass that is enqueued next.
 *   SGR_STAGE_CHUNK_DONE + c    chunk c of the per-Gaussian pass is enqueued: its rows of every per-Gaussian
 *                               output are final on `stream`; the caller can start reducing them while the
 *                               next chunk is computed.
 * num_chunks (<= 1: one) splits the per-Gaussian pass into Gaussian ranges; sgr_backward_chunk_range() gives
 * the range [p0, p1) of a chunk.
 * reduce_records (optional, f32[P,11]): when non-NULL the pass writes (dL_dmeans3D 3 | dL_dopacity 1 |
 * dL_dscales 3 | dL_drotations 4) of Gaussian i as ONE 44-byte record there INSTEAD of the four arrays
 * (whose pointers are then ignored), so that a chunk's all-reduce is one contiguous range;
 * sgr_view_grad_finalize() splits the reduced records back into the arrays. */
#define SGR_STAGE_BLEND_DONE 1
#define SGR_STAGE_CHUNK_DONE 16
typedef void (*SgrStageHook)(void *ctx, int32_t stage);
typedef struct SgrPeerPlan SgrPeerPlan;
typedef struct SgrBackwardPlan {
    SgrStageHook hook; /* may be NULL */
    void *hook_ctx;
    int32_t num_chunks;
    float *reduce_records; /* may be NULL */
    float *dL_dsh_rest;    /* raw-parameter mode (SgrGaussians.activations): f32[P,M-1,3], fully written */
    int32_t chunk_taper;   /* 0: equal chunks; else every chunk half the size of the one before it */
    const SgrPeerPlan *peer; /* NULL: no peer exchange, see SgrPeerPlan below */
} SgrBackwardPlan;
SGR_API int sgr_rasterize_backward_staged(const SgrView *view, const SgrGaussians *g, const int32_t *radii,
                                          const void *geom_buffer, const void *binning_buffer, const void *image_buffer,
                                          int64_t num_rendered, const float *dL_dout_color, float *dL_dmeans2D,
                                          float *dL_dcolors, float *dL_dopacity, float *dL_dmeans3D, float *dL_dcov3D,
                                          float *dL_dsh, float *dL_dscales, float *dL_drotations, void *grad_scratch,
                                          void *stream, const SgrBackwardPlan *plan);
SGR_API int sgr_backward_chunk_range(int32_t P, int32_t num_chunks, int32_t chunk, int32_t taper, int32_t *p0,
                                     int32_t *p1); /* taper: SgrBackwardPlan.chunk_taper */

/* Epilogue of the view-parallel step for the Gaussians [p0, p1), after the exchange (either half optional):
 *  - dL_dsh[P,M,3] rows = sum over views v of basis_k(normalize(mean - campos[v])) * dRGB[v][P,3]  (the SH part of
 *    backward.cu:20-139 is an outer product per view): the gathered factors of view v start at dRGB + v * view_stride
 *    floats (f32[P,3]; view_stride >= 3P) and its camera position at campos + v * campos_stride floats -- the
 *    exchange appends every view's camera position to its factor block so that one all-gather carries both;
 *  - reduced_records f32[P,11] (all-reduced) are split into dL_dmeans3D / dL_dopacity / dL_dscales / dL_drotations.
 * Every output row of the range is fully written; `scale` (e.g. 1/num_views) multiplies everything. */
SGR_API int sgr_view_grad_finalize(int32_t P, int32_t p0, int32_t p1, int32_t M, int32_t sh_degree, int32_t num_views,
                                   const float *means3D, const float *campos, const float *dRGB, int64_t view_stride,
                                   int32_t campos_stride, float *dL_dsh, const float *reduced_records, float scale,
                                   float *dL_dmeans3D, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                                   void *stream);

/* ---- View-parallel exchange over peer memory (NVLink / NVSwitch): csrc/sgr_peer.cu.  No counterpart in the reference.
 * sgr_peer_alloc     one zero-filled device allocation on the current device whose CUDA IPC handle (sgr_peer_export,
 *                    64 bytes, to be sent to the other ranks by any means) maps it at offset 0;
 * sgr_peer_import    maps a peer's allocation into this process (lazy peer access); sgr_peer_close unmaps it.
 * Flag words: the first sgr_peer_flag_bytes() of an allocation used with signal / wait are u32
 * [SGR_PEER_MAX_SLOTS][SGR_PEER_MAX_RANKS]; word [slot][j] is written by rank j only.
 * sgr_peer_signal    (on `stream`) writes `seq` into word [slot][my_rank] of EVERY rank's flags (flag_tab: device array
 *                    of nranks pointers to the ranks' flag words), after a system-scope fence;
 * sgr_peer_wait      (on `stream`) spins until words [slot0 .. slot0+nslots)[0 .. nranks) of the LOCAL flags have all
 *                    reached seq (wrap-safe); traps after timeout_s seconds (<= 0: 20 s) instead of hanging;
 * sgr_peer_reduce_records_synced  second half of the records' all-reduce for the chunk of Gaussians [p0, p1) (p0 a
 *                    multiple of 64): this rank sums the slice of the chunk it OWNS -- the 64-record blocks b with
 *                    b * nranks / blocks == my_rank, the ones the per-Gaussian pass stored here
 *                    (SgrPeerPlan.peer_record_stages) -- over the nranks staging arrays rec_tab points to (device
 *                    array of pointers to f32[11P + 4]; normally all LOCAL), in rank order, and stores the sums into
 *                    every rank's sum array (sum_tab, likewise; remote entries are posted NVLink writes).  The flag
 *                    handshake is folded into the kernel: it first waits until every rank's word of wait_slot in the
 *                    LOCAL flags has reached seq (flags NULL: no wait), and its last CTA to finish writes seq into
 *                    word [signal_slot][my_rank] of every rank's flags (flag_tab NULL: no signal; `counter`: a
 *                    zero-initialised u32 in local device memory that the kernel re-arms, one per concurrently running
 *                    launch). */
#define SGR_PEER_MAX_RANKS 64
#define SGR_PEER_MAX_SLOTS 64
SGR_API int sgr_peer_alloc(size_t bytes, void **ptr);
SGR_API int sgr_peer_free(void *ptr);
SGR_API int sgr_peer_export(const void *ptr, void *handle64);
SGR_API int sgr_peer_import(const void *handle64, void **ptr);
SGR_API int sgr_peer_close(void *ptr);
SGR_API size_t sgr_peer_flag_bytes(void);
SGR_API int sgr_peer_signal(void *const *flag_tab, int32_t nranks, int32_t slot, int32_t my_rank, uint32_t seq,
                            void *stream);
SGR_API int sgr_peer_wait(const void *flags, int32_t nranks, int32_t slot0, int32_t nslots, uint32_t seq,
                          double timeout_s, void *stream);
SGR_API int sgr_peer_reduce_records_synced(const void *const *rec_tab, void *const *sum_tab, int32_t nranks,
                                           int32_t my_rank, int32_t p0, int32_t p1, const void *flags, int32_t wait_slot,
                                           void *const *flag_tab, int32_t signal_slot, uint32_t seq, void *counter,
                                           double timeout_s, void *stream);

/* The peer exchange of a backward (SgrBackwardPlan.peer): the backward signals the peer ranks itself, on `stream`,
 * with sequence number peer_seq: slot peer_slot_blend once the blend pass is enqueued (dL_dcolors, which the caller
 * placed in its peer-visible factor block, is final), slot peer_slot_chunk0 + c after chunk c of the per-Gaussian
 * pass (reduce_records, placed in the peer-visible record array, holds the chunk's rows).  The backward checks every
 * field before it enqueues anything. */
struct SgrPeerPlan {
    void *const *peer_flag_tab; /* DEVICE array of peer_nranks pointers: every rank's flag words, see sgr_peer_signal */
    int32_t peer_nranks, peer_rank, peer_slot_blend, peer_slot_chunk0;
    uint32_t peer_seq;
    /* With SH colours and dL_dsh non-NULL: peer_view_blocks is a DEVICE array of peer_nranks pointers to the ranks'
     * factor blocks (f32[3P] dL/dRGB followed by the rank's camera position; entry peer_rank is dL_dcolors itself).
     * The backward then waits (on `stream`, through peer_flags = this rank's own flag words) until every rank has
     * signalled peer_slot_blend, and the per-Gaussian pass writes dL_dsh = peer_dsh_scale * SUM over all ranks' views
     * of their SH gradients, loading the other ranks' factors straight from their memory -- the all-gather of the
     * factors is fused into the kernel and no separate SH epilogue runs. */
    const float *const *peer_view_blocks;
    const void *peer_flags;
    float peer_dsh_scale;
    double peer_timeout_s;
    /* With peer_view_blocks: DEVICE array of peer_nranks pointers, entry j = rank j's staging array (f32[11P + 4]) for
     * records COMING FROM this rank (entry peer_rank = reduce_records itself).  CTA b of a chunk's launch then stores its
     * 64 records into the array of the rank that owns them (owner = b * nranks / CTAs of the chunk; what
     * sgr_peer_reduce_records_synced assumes) with a TMA bulk store over NVLink -- the reduce-scatter half of the
     * records' all-reduce is fused into the pass.  NULL: all records go to reduce_records. */
    float *const *peer_record_stages;
    /* Optional second stream for the backward's own signals: each signal kernel then runs there, behind an event
     * recorded on `stream`, and the per-Gaussian chunks follow one another on `stream` without the signals' launches
     * in between.  The caller orders whatever must see the signals' completion behind this stream. */
    void *peer_signal_stream;
    /* Optional: the backward also drives the records' exchange, on this side stream, chunk by chunk underneath the
     * per-Gaussian pass of the later chunks: once this rank's CHUNK c signal is out (an event behind the signal kernel;
     * a spinning kernel must never sit in front of a signal another rank waits for) it enqueues
     * sgr_peer_reduce_records_synced (wait CHUNK c of every rank, sum the owned slice over peer_rec_tab into every rank's
     * peer_sum_tab, signal peer_slot_reduced0 + c) and, behind the NEXT chunk's reduce, sgr_peer_wait(REDUCED c) + the
     * split of peer_sums (this rank's sum array) into dL_dmeans3D / dL_dopacity / dL_dscales / dL_drotations scaled by
     * peer_dsh_scale.  The caller orders its stream behind peer_side_stream (and peer_signal_stream) afterwards.
     * peer_emulate_ranks (tests): bit r set = also reduce rank r's slices here. */
    void *peer_side_stream;
    const void *const *peer_rec_tab;
    void *const *peer_sum_tab;
    const float *peer_sums;
    int32_t peer_slot_reduced0;
    uint64_t peer_emulate_ranks;
};

/* markVisible (rasterizer_impl.cu:141-153): present[i] = view-space z > 0.2. */
SGR_API int sgr_mark_visible(int32_t P, const float *means3D, const float *viewmatrix,
                     const float *projmatrix, uint8_t *present, void *stream);

/* Sizes of the opaque buffers (what `required<T>(P)` is in rasterizer_impl.h:66-72). */
SGR_API size_t sgr_geometry_bytes(int32_t P);
SGR_API size_t sgr_binning_bytes(int64_t capacity);
SGR_API size_t sgr_image_bytes(int32_t width, int32_t height);
SGR_API size_t sgr_backward_scratch_bytes(int32_t P);

/* Decode the opaque buffers into the reference's named arrays, for parity tests
 * (GeometryState / BinningState / ImageState, rasterizer_impl.h:30-63).  Any output may be NULL.
 *   depths f32[P], means2D f32[P,2], conic_opacity f32[P,4], rgb f32[P,3], clamped u8[P,3],
 *   tiles_touched u32[P]; keys u64[R] = (tile<<32 | depth bits) in sorted order,
 *   point_list u32[R]; ranges u32[T,2]; final_T f32[H,W]; n_contrib u32[H,W];
 *   footprint u8[R]: per sorted instance, which of its tile's eight 8x4-pixel blocks (bit = band*2 + half)
 *   the splat can reach with alpha >= 1/255 -- this library's own culling state, not a reference array
 *   (0xff when the list carries no masks, i.e. P > 2^24). */
SGR_API int sgr_inspect_state(int32_t P, int32_t width, int32_t height, int64_t num_rendered,
                      const void *geom_buffer, const void *binning_buffer, const void *image_buffer,
                      float *depths, float *means2D, float *conic_opacity, float *rgb, uint8_t *clamped,
                      uint32_t *tiles_touched, uint64_t *keys, uint32_t *point_list, uint32_t *ranges,
                      float *final_T, uint32_t *n_contrib, uint8_t *footprint, void *stream);

/* ------------------------------------------------------------------------------------------
 * SuGaR surface-regularisation field: fused K-neighbour gather + anisotropic density / SDF.
 * Replaces the PyTorch ops of SuGaR.get_field_values (sugar_model.py:1247-1316, beta_mode
 * 'average' sugar_model.py:1192-1195) and SuGaR.compute_density (:1345-1368).
 *   x          f32[N,3]   sample points
 *   nbr_idx    i64[N,K]   neighbour Gaussian indices per sample (knn_idx[gaussian_idx])
 *   points f32[P,3], scaling f32[P,3] (activated), quaternions f32[P,4] (normalised, w first),
 *   strengths f32[P] (sigmoid(densities))
 * Outputs (any may be NULL): density f32[N] (before the straight-through clamp),
 *   nbr_opacity f32[N,K], beta f32[N], sdf f32[N].
 * ------------------------------------------------------------------------------------------ */
typedef struct SgrFieldParams {
    int32_t N, K, P;
    float density_factor;
    float density_threshold;
    float opacity_min_clamp; /* 1e-16 in the reference */
    int32_t samples_per_idx_row; /* 0/1: nbr_idx is i64[N,K]; g > 1: i64[ceil(N/g),K], row n/g serves sample n
                                  * (ray samples that share their pixel's neighbours, sugar_model.py:1980) */
} SgrFieldParams;

/* `scratch` must hold sgr_field_scratch_bytes(P) (packed per-Gaussian records; device memory). */
SGR_API size_t sgr_field_scratch_bytes(int32_t P);

SGR_API int sgr_field_forward(const SgrFieldParams *p, const float *x, const int64_t *nbr_idx,
                      const float *points, const float *scaling, const float *quaternions,
                      const float *strengths,
                      float *density, float *nbr_opacity, float *beta, float *sdf,
                      void *scratch, void *stream);

/* Backward of the above.  Upstream grads (any may be NULL = zero): g_density f32[N],
 * g_nbr_opacity f32[N,K], g_beta f32[N], g_sdf f32[N].  Downstream grads are fully WRITTEN
 * (any may be NULL): g_x f32[N,3], g_points f32[P,3], g_scaling f32[P,3],
 * g_quaternions f32[P,4] (w.r.t. the quaternion passed in, through two_s = 2/|q|^2 exactly as
 * pytorch3d's quaternion_to_matrix differentiates), g_strengths f32[P]. */
SGR_API int sgr_field_backward(const SgrFieldParams *p, const float *x, const int64_t *nbr_idx,
                       const float *points, const float *scaling, const float *quaternions,
                       const float *strengths,
                       const float *g_density, const float *g_nbr_opacity, const float *g_beta,
                       const float *g_sdf,
                       float *g_x, float *g_points, float *g_scaling, float *g_quaternions,
                       float *g_strengths, void *scratch, void *stream);

/* Density estimation loss of the coarse_density trainer in projection mode
 * (sugar_trainers/coarse_density.py:654-656, 684-691), per sample n drawn from Gaussian g = own_idx[n]:
 *   rho  = sgr_field_forward's density at x_n (before the straight-through clamp), beta its beta
 *   e    = <x_n - points[g], n_g>,  n_g = column argmin_j scaling[g][j] of R(quaternions[g]) (first minimum)
 *   loss[n] = | rho - exp(-0.5 e^2 / beta^2) |
 * Same arguments as sgr_field_forward plus own_idx i64[N]; p->samples_per_idx_row must be 0 or 1 and
 * density_threshold / opacity_min_clamp are not used.  loss f32[N] is required, nbr_opacity f32[N,K] may be
 * NULL and equals sgr_field_forward's.  `scratch` must hold sgr_field_scratch_bytes(P).
 * Backward: g_loss f32[N] -> g_x, g_points, g_scaling, g_quaternions, g_strengths as in sgr_field_backward
 * (fully written, any may be NULL); no gradient flows through the argmin. */
SGR_API int sgr_density_estimation_forward(const SgrFieldParams *p, const float *x, const int64_t *own_idx,
                                           const int64_t *nbr_idx, const float *points, const float *scaling,
                                           const float *quaternions, const float *strengths, float *loss,
                                           float *nbr_opacity, void *scratch, void *stream);
SGR_API int sgr_density_estimation_backward(const SgrFieldParams *p, const float *x, const int64_t *own_idx,
                                            const int64_t *nbr_idx, const float *points, const float *scaling,
                                            const float *quaternions, const float *strengths, const float *g_loss,
                                            float *g_x, float *g_points, float *g_scaling, float *g_quaternions,
                                            float *g_strengths, void *scratch, void *stream);

/* ------------------------------------------------------------------------------------------
 * "Better normal" regularisation of the trainers (sugar_trainers/coarse_sdf.py:688-716, with
 * SuGaR.get_normals(estimate_from_points=False) -> get_smallest_axis, sugar_model.py:930-968), in the
 * trainers' only mode sdf_better_normal_gradient_through_normal_only=True (weights and signs detached):
 *   n_g = column argmin_j scaling[g][j] of R(quaternions[g]);  m_k = sign(<n_k, n_own>) n_k
 *   w_k = nbr_opacity[n,k] |<x_n - mu_k, m_k>| / max(min_j scaling[k][j], 1e-6)^2, / max(sum_k w_k, 1e-6)
 *   loss[n] = | n_own - sum_k w_k m_k |^2
 * Inputs: x f32[N,3], own_idx i64[N] (sdf_gaussian_idx), nbr_idx i64[N,K] (knn_idx[own_idx]),
 * points/scaling f32[P,3], quaternions f32[P,4], nbr_opacity f32[N,K] (fields['closest_gaussian_opacities']).
 * Backward: g_loss f32[N] -> g_quaternions f32[P,4], fully written (the only differentiable input).
 * `scratch` must hold sgr_normal_scratch_bytes(P).
 * ------------------------------------------------------------------------------------------ */
SGR_API size_t sgr_normal_scratch_bytes(int32_t P);
SGR_API int sgr_normal_loss_forward(int32_t N, int32_t K, int32_t P, const float *x, const int64_t *own_idx,
                                    const int64_t *nbr_idx, const float *points, const float *scaling,
                                    const float *quaternions, const float *nbr_opacity, float *loss, void *scratch,
                                    void *stream);
SGR_API int sgr_normal_loss_backward(int32_t N, int32_t K, int32_t P, const float *x, const int64_t *own_idx,
                                     const int64_t *nbr_idx, const float *points, const float *scaling,
                                     const float *quaternions, const float *nbr_opacity, const float *g_loss,
                                     float *g_quaternions, void *scratch, void *stream);

/* ------------------------------------------------------------------------------------------
 * Gaussians bound to a triangle mesh (refinement stage): the property code of a bound SuGaR model,
 * sugar_scene/sugar_model.py:384-398 (points), :415-441 (scaling), :443-479 (quaternions), as one kernel
 * and its backward.  F faces, n_per Gaussians per face (P = F * n_per), V vertices.
 *   verts f32[V,3], faces i64[F,3], bary f32[n_per,3] (surface_triangle_bary_coords, device memory),
 *   scales_raw f32[P,2] (_scales: log of the two in-plane scales), complex_raw f32[P,2] (_quaternions: the
 *   learned in-plane rotation as a complex number, normalised here), thickness = surface_mesh_thickness.
 * Outputs, fully written: points f32[P,3], scaling f32[P,3] = (thickness, exp, exp), quaternions f32[P,4]
 * (normalised, w first; pytorch3d 0.7.4 matrix_to_quaternion of [normal | rotated edge | cross]).
 * Backward: g_verts f32[V,3] (zeroed here, then accumulated), g_scales_raw, g_complex_raw f32[P,2] fully written.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_meshbind_forward(int32_t F, int32_t n_per, int32_t V, const float *verts, const int64_t *faces,
                                 const float *bary, const float *scales_raw, const float *complex_raw, float thickness,
                                 float *points, float *scaling, float *quaternions, void *stream);
SGR_API int sgr_meshbind_backward(int32_t F, int32_t n_per, int32_t V, const float *verts, const int64_t *faces,
                                  const float *bary, const float *scales_raw, const float *complex_raw,
                                  const float *g_points, const float *g_scaling, const float *g_quaternions,
                                  float *g_verts, float *g_scales_raw, float *g_complex_raw, void *stream);

/* The editable bound model (make_editable / get_edited_quaternions_and_scales, sugar_model.py:562-667, and the
 * `scaling` / `quaternions` properties with editable set), forward only: the forward above at the current `verts`,
 * with each Gaussian's in-plane rotation turned by the bary-weighted change in angle of its face's vertex axes and
 * each plane scale multiplied by the bary-weighted stretch of those axes, both measured against `reference_verts`
 * f32[V,3] (the vertices make_editable snapshotted).  out_rows NULL: Gaussian g goes to row g of points / scaling /
 * quaternions; else to row out_rows[g] (i64[P]), and a negative entry skips it. */
SGR_API int sgr_meshbind_edited_forward(int32_t F, int32_t n_per, int32_t V, const float *verts,
                                        const float *reference_verts, const int64_t *faces, const float *bary,
                                        const float *scales_raw, const float *complex_raw, float thickness,
                                        const int64_t *out_rows, float *points, float *scaling, float *quats,
                                        void *stream);

/* ------------------------------------------------------------------------------------------
 * SH colours at a rotated view direction (SuGaRCompositor's sh_rotations, sugar_compositor.py:139-151):
 * colors[i] = max(eval_sh(normalize(means[i] - campos) @ R_g) + 0.5, 0) per channel, in the rasterizer's own basis
 * and rounding (at R = I the forward's in-kernel colour, to the bit).  Rows group_start[g] .. group_start[g+1] - 1
 * (i64[G+1], group_start[0] = 0, group_start[G] = P) take group_rot[g] (f32[G,9], row-major 3x3).
 *   means f32[P,3], shs f32[P,M,3] with (sh_degree + 1)^2 <= M, campos f32[3], colors f32[P,3].  Forward only.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_sh_colors_rotated(int32_t P, int32_t M, int32_t sh_degree, const float *means, const float *shs,
                                  const float *campos, int32_t G, const int64_t *group_start, const float *group_rot,
                                  float *colors, void *stream);

/* ------------------------------------------------------------------------------------------
 * Exact K-nearest-neighbour search (uniform grid).  Replaces pytorch3d.ops.knn_points as SuGaR
 * calls it: reset_neighbors (sugar_model.py:1013-1030, queries == points, K = 16) and
 * get_gaussians_closest_to_samples (sugar_model.py:1335-1343).
 *   points f32[P,3] reference cloud, queries f32[Q,3]; 0 < K <= min(P, 64)
 *   idx i64[Q,K], dist2 f32[Q,K]: neighbours ordered by increasing squared distance.
 * `workspace` must hold sgr_knn_workspace_bytes(P).
 * ------------------------------------------------------------------------------------------ */
SGR_API size_t sgr_knn_workspace_bytes(int32_t P);
SGR_API int sgr_knn(int32_t P, const float *points, int32_t Q, const float *queries, int32_t K, int64_t *idx,
                    float *dist2, void *workspace, void *stream);

/* ------------------------------------------------------------------------------------------
 * distCUDA2 (simple-knn, called by GaussianModel.create_from_pcd, gaussian_model.py:134): per point of
 * points f32[P,3], mean_dist2 f32[P] <- (b0 + b1 + b2) / 3 of its three smallest squared distances to OTHER points
 * (by index: a duplicate position counts as 0), each distance rounded as the reference build rounds it, so the result
 * is the reference's to the bit.  P <= 3 keeps the reference's FLT_MAX sentinels in the sum: inf for P <= 2,
 * (b0 + b1 + FLT_MAX) / 3 for P = 3.  The search is sgr_knn's cell grid, so `workspace` is the same buffer:
 * sgr_knn_workspace_bytes(P) bytes.  P = 0 does nothing.  No host synchronisation.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_dist_cuda2(int32_t P, const float *points, float *mean_dist2, void *workspace, void *stream);

/* ------------------------------------------------------------------------------------------
 * Photometric loss of the trainers, (1 - f) * l1_loss + f * (1 - ssim) (sugar_utils/loss_utils.py:17-62, used as
 * sugar_trainers/coarse_sdf.py:101-103, 452-457): per image b of img1, img2 f32[B,C,H,W] (contiguous planes), the
 * mean over its C*H*W elements of |x - y| and of the SSIM map
 *   S = (2 mu1 mu2 + c1)(2 sigma12 + c2) / ((mu1^2 + mu2^2 + c1)(sigma1^2 + sigma2^2 + c2))
 * whose moments are 11x11 windowed sums with zero padding of 5, each (b, c) plane on its own.  The window is
 * window[i] * window[j] (passed by value: the caller builds the 1-D weights by its recipe).
 *   partial_maps  f32[3, B*C*H*W]  the op's saved state: dS/dmu1 (sigma1^2, sigma12 expanded), dS/dE[x^2], dS/dE[xy]
 *   per_image_out f32[B, 2]        (l1 mean, ssim mean) per image, summed in a fixed order (run-to-run identical)
 *   scratch       sgr_l1_ssim_scratch_bytes(B, C, H, W) bytes of device memory
 * Backward: g_l1, g_ssim f32[B] (DEVICE: the upstream gradients of the two outputs) -> grad_img1 f32[B,C,H,W], fully
 * written; only img1 is differentiated (sign(0) = 0 for the L1 term).  Limits: B*C*H*W <= 2^31 - 1, B*C <= 65535.
 * ------------------------------------------------------------------------------------------ */
typedef struct SgrSsimParams {
    int32_t B, C, H, W;
    float c1, c2;      /* 0.01^2, 0.03^2 in the reference */
    float window[11];  /* normalised 1-D weights */
} SgrSsimParams;
SGR_API size_t sgr_l1_ssim_scratch_bytes(int32_t B, int32_t C, int32_t H, int32_t W);
SGR_API int sgr_l1_ssim_forward(const SgrSsimParams *p, const float *img1, const float *img2, float *partial_maps,
                                float *per_image_out, void *scratch, void *stream);
SGR_API int sgr_l1_ssim_backward(const SgrSsimParams *p, const float *img1, const float *img2, const float *partial_maps,
                                 const float *g_l1, const float *g_ssim, float *grad_img1, void *stream);

/* ------------------------------------------------------------------------------------------
 * Mesh normal consistency of the refinement stage (sugar_trainers/refine.py:775-783: pytorch3d 0.7.4
 * mesh_normal_consistency of the one surface mesh): the mean over the Q pairs of faces that share an edge of
 *   1 - cosine_similarity(n_a, -n_b, eps = 1e-8),  n_x = (verts[v1] - verts[v0]) x (verts[x] - verts[v0])
 * over a pair table built once per topology (sugar_b200/meshloss.py: mesh_topology):
 *   verts    f32[V,3]
 *   pairs    i32[Q,4]   rows (v0, v1, a, b): the shared edge (v0 < v1) and the two faces' opposite vertices
 *   vert_ptr i32[V+1], vert_inc i32[4Q]   for each vertex, the entries 4 q + slot of `pairs` that name it, in
 *                                          ascending order (CSR)
 *   loss     f32[1]     the mean; summed in a fixed order (run-to-run identical); Q = 0 gives 0 (a memset only)
 * The per-pair arithmetic is in double; where both normals are longer than eps the term is evaluated as
 * |n_a/|n_a| + n_b/|n_b||^2 / 2, which keeps its digits at small angles.
 * Backward: g_loss f32[1] (DEVICE: the upstream gradient) -> g_verts f32[V,3], fully written, each vertex summed
 * over its CSR list in order (run-to-run identical).  Limits: 0 <= Q <= (2^31 - 1) / 4.
 * ------------------------------------------------------------------------------------------ */
SGR_API size_t sgr_mesh_nc_forward_scratch_bytes(int32_t Q);
SGR_API size_t sgr_mesh_nc_backward_scratch_bytes(int32_t Q);
SGR_API int sgr_mesh_nc_forward(int32_t Q, int32_t V, const float *verts, const int32_t *pairs, float *loss,
                                void *scratch, void *stream);
SGR_API int sgr_mesh_nc_backward(int32_t Q, int32_t V, const float *verts, const int32_t *pairs,
                                 const int32_t *vert_ptr, const int32_t *vert_inc, const float *g_loss, float *g_verts,
                                 void *scratch, void *stream);

/* ------------------------------------------------------------------------------------------
 * Mesh Laplacian smoothing of the refinement stage (sugar_trainers/refine.py:163-171, 778-780: pytorch3d 0.7.4
 * mesh_laplacian_smoothing of the one surface mesh, off by default there): loss = sum_v |y_v| / V over every vertex,
 *   uniform  y = L x                                L[i,j] = 1 / deg_i per unique-edge entry, L[i,i] -= 1
 *   cot      y = (L x) norm_w - x                   L the cotangent Laplacian, norm_w = 1 / rowsum(L) where > 0
 *   cotcurv  y = (L x - rowsum(L) x) 0.25 inv_area  inv_area = 1 / (the areas of the faces on v) where > 0, else 0
 * L is a constant (no gradient through it), computed from a topology built once (sugar_b200/meshloss.py:
 * laplacian_topology):
 *   verts    f32[V,3]
 *   faces    i32[F,3]                          (cot / cotcurv; not read for uniform)
 *   vert_ptr i32[V+1], vert_inc               uniform: the neighbours of each vertex, i32[2E] over the E unique
 *                                              edges, a self-loop (v, v) listed twice; cot / cotcurv: the entries
 *                                              3 f + k of the face corners at each vertex, i32[3F]; ascending (CSR)
 *   face_w   f32[F,4]   (cot / cotcurv) written by the forward, read by the backward: (cot_a, cot_b, cot_c) / 4 and
 *                        the clamped Heron area of each face, in pytorch3d's float32 order
 *   vert_ys  f32[V,4]   written by the forward, read by the backward: y_v and the row's scale (1 / deg, norm_w or
 *                        0.25 inv_area)
 *   partials f64[SGR_MESH_LAP_PARTIALS]   scratch
 *   loss     f32[1]     the mean; summed in double in a fixed order (run-to-run identical)
 * Backward: g_loss f32[1] (DEVICE: the upstream gradient) -> g_verts f32[V,3], fully written; each vertex gathers its
 * CSR list in order (run-to-run identical); rows with y_v = 0 contribute no gradient.  No host synchronisation.
 * Limits: V > 0, 0 < F <= (2^31 - 1) / 3.
 * ------------------------------------------------------------------------------------------ */
#define SGR_MESH_LAP_UNIFORM 0
#define SGR_MESH_LAP_COT 1
#define SGR_MESH_LAP_COTCURV 2
#define SGR_MESH_LAP_PARTIALS 1024
SGR_API int sgr_mesh_lap_forward(int32_t method, int32_t V, int32_t F, const float *verts, const int32_t *faces,
                                 const int32_t *vert_ptr, const int32_t *vert_inc, float *face_w, float *vert_ys,
                                 double *partials, float *loss, void *stream);
SGR_API int sgr_mesh_lap_backward(int32_t method, int32_t V, int32_t F, const int32_t *faces, const int32_t *vert_ptr,
                                  const int32_t *vert_inc, const float *face_w, const float *vert_ys,
                                  const float *g_loss, float *g_verts, void *stream);

/* ------------------------------------------------------------------------------------------
 * Border-face erosion of the refined mesh (postprocess_mesh, sugar_extractors/refined_mesh.py:140-147): `iterations`
 * rounds, each one launch on `stream`, no host synchronisation.  Entry 3 f + m is edge m of face f, (0,1), (1,2),
 * (2,0); the entries are grouped in runs of equal (unordered) edges, built once per call by the caller
 * (sugar_b200/postprocess.py):
 *   entry_run i32[3F]    the run of each entry
 *   run_ptr   i32[R+1]   CSR offsets of the runs into run_faces (entries past R are not read)
 *   run_faces i32[3F]    the face of each entry, run by run
 *   mask      u8[F]      in: the live faces (0 / 1); out: those alive after the rounds
 *   mask_tmp  u8[F]      scratch, distinct from mask
 * A live face stays in a round iff each of its three runs holds at least 2 entries whose face was live at the start
 * of the round (a face's own two entries on one edge count twice).  Deterministic, no atomics.
 * Limits: 0 <= F <= (2^31 - 1) / 3, iterations >= 0.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_border_peel(int32_t F, int32_t iterations, const int32_t *entry_run, const int32_t *run_ptr,
                            const int32_t *run_faces, uint8_t *mask, uint8_t *mask_tmp, void *stream);

/* ------------------------------------------------------------------------------------------
 * Splatted mesh and nearest-face triangle z-buffer: the default depth source of the level-set extraction
 * (compute_level_surface_points_from_camera_fast with use_gaussian_depth=False, sugar_model.py:1880-1968).
 * sgr_splat_mesh: SuGaR.splat_mesh(camera) for primitive 'diamond', mode 'perspective' (sugar_model.py:481-514,
 * 695-728): four vertices per Gaussian, mu -/+ t s_a1 R[:,a1], mu +/- t s_a2 R[:,a2] (a0 = argmin s, lowest index on
 * ties; a1, a2 the next two axes cyclically; t = triangle_scale; vertex order (-a1, +a2, +a1, -a2)), each moved along
 * its view ray onto the plane through the centre perpendicular to the centre's ray.
 *   points f32[P,3], scaling f32[P,3] (activated), quaternions f32[P,4] (w first; 16-byte aligned),
 *   viewmatrix f32[16] (the rasterizer's transposed world->view), view_inverse f32[16] (its inverse, same layout),
 *   verts f32[4P,3] (16-byte aligned), fully written.  The arithmetic is in double.  P = 0 launches nothing.
 * sgr_mesh_raster: pytorch3d 0.7.4 MeshRasterizer (blur_radius 0, perspective-correct, no culling) read at its first
 * face per pixel, for any mesh verts f32[V,3], faces i64[F,3] (ids outside [0, V) make the face cover nothing):
 * vertices through viewmatrix (view z) and projmatrix (/ (w + 1e-7)), pixel (i, j) sampled at the rasterizer's ndc
 * (2i+1)/W - 1; a face covers a pixel when every perspective-corrected barycentric is > 0 and the depth pz >= 0, and
 * the pixel keeps the face of least pz (equal pz: the lower face id).  Unlike pytorch3d's binned path the result is
 * complete however many faces overlap one region.
 *   zbuf f32[H,W] (pz, -1 where no face covers), pix_to_face i64[H,W] (-1 there), fully written; identical from run to
 *   run.  Limits: W, H <= 65535, W*H <= 2^31 - 1.  `scratch`: sgr_mesh_raster_scratch_bytes(F, W, H) bytes.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_splat_mesh(int32_t P, const float *points, const float *scaling, const float *quaternions,
                           const float *viewmatrix, const float *view_inverse, float triangle_scale, float *verts,
                           void *stream);
SGR_API size_t sgr_mesh_raster_scratch_bytes(int32_t F, int32_t W, int32_t H);
SGR_API int sgr_mesh_raster(int32_t V, int32_t F, const float *verts, const int64_t *faces, const float *viewmatrix,
                            const float *projmatrix, int32_t W, int32_t H, float *zbuf, int64_t *pix_to_face,
                            void *scratch, void *stream);

/* ------------------------------------------------------------------------------------------
 * UV texture of a mesh with n Gaussians bound per face (extract_texture_image_and_uv_from_gaussians,
 * sugar_model.py:2464-2677, n_sh 1, texture_with_gaussian_renders).  The layout: square size s >= 3,
 * n_sq = int(sqrt(F / 2 + 1) + 1), T = s * n_sq; square k = (k / n_sq, k % n_sq) holds face 2k (bottom) and 2k + 1 (top).
 * sgr_texture_init: the initial texels, float32 as the reference computes them.  Every texel a face owns takes
 * SH2RGB(sh_dc) of the face's Gaussian (f*n ... f*n + n-1) of greatest density at the texel's fixed barycentric point
 * (torch argmax: NaN first, ties to the first); every other texel is 0.5.
 *   verts f32[V,3], faces i64[F,3] (a face with an id outside [0, V) owns no texel), points / scaling f32[F*n,3],
 *   quaternions f32[F*n,4] (w first; 16-byte aligned), sh_dc f32[F*n,3], texture f32[T,T,3] fully written.
 *   T must equal the layout's; T*T <= 2^31 - 1.
 * sgr_texture_bake_view: one view of the bake.  Every pixel with pix_to_face >= 0 and zbuf > 0 finds its texel
 * (perspective-correct barycentrics in double through the z-buffer's projection, UV interpolated in float32, TexturesUV's
 * nearest lookup); per texel, the pixel of highest row-major index adds clamp(image, 0, 1) to tex_sum and 1 to
 * tex_count.  No float atomics: the sums are identical from run to run.
 *   verts_uv f32[n_uv,2] (8-byte aligned), faces_uv i64[F,3], image f32[3,H,W], zbuf f32[H,W], pix_to_face i64[H,W]
 *   (values outside [0, F) are empty pixels), tex_sum f32[T,T,3], tex_count i32[T,T] (accumulated), owner i32[T,T]
 *   (all -1 on entry and on return), pix_texel i32[H,W] scratch.  T*T, W*H <= 2^31 - 1.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_texture_init(int32_t F, int32_t n, int32_t V, int32_t square_size, int32_t T, const float *verts,
                             const int64_t *faces, const float *points, const float *scaling, const float *quaternions,
                             const float *sh_dc, float *texture, void *stream);
SGR_API int sgr_texture_bake_view(int32_t V, int32_t F, int32_t n_uv, int32_t T, const float *verts,
                                  const int64_t *faces, const float *verts_uv, const int64_t *faces_uv,
                                  const float *viewmatrix, const float *projmatrix, int32_t W, int32_t H,
                                  const float *image, const float *zbuf, const int64_t *pix_to_face, float *tex_sum,
                                  int32_t *tex_count, int32_t *owner, int32_t *pix_texel, void *stream);
/* sgr_texture_render: the textured mesh's image as metrics.py renders it (MeshRasterizer, faces_per_pixel 1, blur 0;
 * SoftPhongShader with AmbientLights and default Materials, so the shaded colour is the texel; softmax_rgb_blend with
 * sigma = gamma = 1e-4).  Every pixel with pix_to_face in [0, F) samples `texture` at the face's UV (the bake's
 * barycentrics and float32 UV) as TexturesUV does: grid_sample on the map flipped in y at 2 uv - 1, align_corners,
 * border padding, bilinear (torch's weights and summation order) or nearest; then blends with the K = 1 formula,
 * z_inv = (zfar - zbuf) / (zfar - znear), w = exp((z_inv - max(z_inv, eps)) / gamma), delta = max(exp((eps -
 * max(z_inv, eps)) / gamma), eps), eps = 1e-10, out = (w c + delta bg) / (w + delta).  The edge term prob is taken as
 * 1 (pytorch3d's is sigmoid(-dists / sigma) < 1 near a face's edges).  Other pixels (and faces with a vertex or UV id out
 * of range) are bg.  Deterministic, no atomics.
 *   texture f32[Ht,Wt,3], verts_uv f32[n_uv,2] (8-byte aligned), faces_uv i64[F,3], zbuf f32[H,W], pix_to_face i64[H,W],
 *   sampling_mode SGR_SAMPLE_*, finite znear < zfar, image f32[3,H,W] fully written.  Wt*Ht, W*H <= 2^31 - 1. */
#define SGR_SAMPLE_BILINEAR 0
#define SGR_SAMPLE_NEAREST 1
SGR_API int sgr_texture_render(int32_t V, int32_t F, int32_t n_uv, int32_t Wt, int32_t Ht, const float *verts,
                               const int64_t *faces, const float *verts_uv, const int64_t *faces_uv,
                               const float *texture, const float *viewmatrix, const float *projmatrix, int32_t W,
                               int32_t H, const float *zbuf, const int64_t *pix_to_face, int32_t sampling_mode,
                               float bg_r, float bg_g, float bg_b, double znear, double zfar, float *image,
                               void *stream);

/* ------------------------------------------------------------------------------------------
 * Marching-cubes mesh of the coarse model (the use_marching_cubes branch of coarse_mesh.py:623-714).
 * sgr_density_grid: SuGaR.compute_density (sugar_model.py:1345-1368) at every point (x_axis[i], y_axis[j], z_axis[k])
 * of a torch.meshgrid ('ij'): the exact K nearest Gaussian centres by squared distance (sgr_knn's set and order), summed
 * with sgr_field_forward's arithmetic and order, so a voxel equals sgr_field_forward over sgr_knn's neighbours of the
 * same point.  Voxels strictly inside the box (-e, e)^3, e = exclude_extent compared in float32, are 0 without a search
 * (coarse_mesh.py:698); e <= 0 excludes nothing.
 *   points f32[P,3], scaling f32[P,3] (activated), quaternions f32[P,4] (w first, 16-byte aligned), strengths f32[P],
 *   x_axis f32[Rx], y_axis f32[Ry], z_axis f32[Rz], density f32[Rx,Ry,Rz] fully written.
 *   Limits: 0 < K <= min(P, 64), Rx*Ry*Rz <= 2^30.  `workspace`: sgr_density_grid_workspace_bytes(P) bytes.
 * sgr_mcubes_count / sgr_mcubes_emit: marching cubes at `level` (a corner is inside when (double)value > level) with
 * the generated case table of sgr_mcubes_table.h.  One vertex per grid edge whose ends are on different sides, at
 * lower corner + t along the edge, t = (level - f1) / (f2 - f1) in double, in index space; vertices ordered by the
 * edge's lower voxel (C order), then axis x, y, z; triangles (int64 vertex ids) ordered by cube, then table order.
 * count classifies and scans into `scratch` and returns the totals (one stream synchronisation; more than 2^32 - 1 of
 * either is an error); emit, on the same scratch, volume and level, writes verts f32[n_verts,3] and faces i64[n_faces,3].
 *   volume f32[Rx,Ry,Rz] (C order), Rx*Ry*Rz <= 2^30.  `scratch`: sgr_mcubes_scratch_bytes(Rx, Ry, Rz) bytes.
 * ------------------------------------------------------------------------------------------ */
SGR_API size_t sgr_density_grid_workspace_bytes(int32_t P);
SGR_API int sgr_density_grid(int32_t P, const float *points, const float *scaling, const float *quaternions,
                             const float *strengths, int32_t K, float density_factor, int32_t Rx, int32_t Ry,
                             int32_t Rz, const float *x_axis, const float *y_axis, const float *z_axis,
                             float exclude_extent, float *density, void *workspace, void *stream);
SGR_API size_t sgr_mcubes_scratch_bytes(int32_t Rx, int32_t Ry, int32_t Rz);
SGR_API int sgr_mcubes_count(int32_t Rx, int32_t Ry, int32_t Rz, const float *volume, double level, int64_t *n_verts,
                             int64_t *n_faces, void *scratch, void *stream);
SGR_API int sgr_mcubes_emit(int32_t Rx, int32_t Ry, int32_t Rz, const float *volume, double level, int64_t n_verts,
                            int64_t n_faces, float *verts, int64_t *faces, void *scratch, void *stream);

/* ------------------------------------------------------------------------------------------
 * Screened-Poisson reconstruction on a dense grid (sugar_b200/poisson.py states the discrete problem; restated in
 * oracle/poisson_oracle.py).  A grid is f32[N,N,N] in C order with N = 2^depth; a sample's grid coordinates are
 * g = (p - o) * inv_h - 0.5 in float32.  Every grid and buffer is caller-allocated; no float atomics, so every output
 * is identical from run to run.  One stream; the calls that return a host value synchronise it once.
 * sgr_poisson_bin: each sample goes to the bin of its hat support's lower corner clamp(floor(g), 0, N - 2), bin b
 *   holding binned[starts[b] .. starts[b+1]) (the last bin ending at n) in sample order, each record (gx, gy, gz,
 *   sample id bits), by a stable radix sort.  points f32[n,3], starts u32[N^3], binned f32[n,4]; scratch: keys u32[2n],
 *   records f32[n,4] (binned and records 16-byte aligned), hist u32[256 T] with T = ceil(n / 256), block_sums
 *   u32[(max(N^3, 256 T) + 4095) / 4096 + 1]; n_occupied (host) <- the number of non-empty bins.
 * sgr_poisson_splat: every node gathers from its 8 neighbouring bins (increasing bin index, then sample order):
 *   (starts as sgr_poisson_bin wrote them)
 *   mode 0 out0 = -area * sum_s normals[s] . grad phi(g_s), out1 = alpha * area * sum_s phi(g_s) (attr = normals f32[n,3]);
 *   mode 1 out0 = sum_s phi(g_s); mode 2 out0 = sum_s phi(g_s) attr[s, channel] (attr f32[n,3]).  Outputs f32[N^3].
 * sgr_poisson_coarsen: coarse[I] = the sum of the 8 children of I in fine f32[N^3]; coarse f32[(N/2)^3], N >= 8.
 * sgr_poisson_residual_norm: norm (host) <- |b - A u|_2 for A = coeff * (7-point Neumann stencil) + diag(q);
 *   u == NULL gives |b|_2.  partial f64[1024].
 * sgr_poisson_vcycle: one V(2,2) cycle over levels l = 0 .. depth - 2 (side 2^depth >> l, stencil coefficient 2^l):
 *   u, b, q are HOST arrays of depth - 1 device grids; u[0], b[0], q[0] the system, q[l > 0] its sgr_poisson_coarsen
 *   pyramid; u[l > 0] and b[l > 0] are scratch.  norm (host) <- the fine residual norm after the cycle.
 * sgr_poisson_interpolate: values[s] = trilinear interpolation of grid f32[N^3] at g = points[s * stride + a] * scale
 *   + offset (clamped to the grid); with sum != NULL, sum (host) <- the sum of the values (partial f64[1024]).
 *   values may be NULL when sum is given.
 *   Limits: n > 0, N a power of two in [4, 1024], 3 <= depth <= 10.
 * ------------------------------------------------------------------------------------------ */
SGR_API int sgr_poisson_bin(int32_t n, const float *points, int32_t N, float ox, float oy, float oz, float inv_h,
                            uint32_t *starts, float *binned, uint32_t *keys, float *records, uint32_t *hist,
                            uint32_t *block_sums, int64_t *n_occupied, void *stream);
SGR_API int sgr_poisson_splat(int32_t N, int32_t n, const uint32_t *starts, const float *binned, int32_t mode,
                              const float *attr, int32_t channel, float area, float alpha, float *out0, float *out1,
                              void *stream);
SGR_API int sgr_poisson_coarsen(int32_t N, const float *fine, float *coarse, void *stream);
SGR_API int sgr_poisson_residual_norm(int32_t N, float coeff, const float *u, const float *b, const float *q,
                                      double *partial, double *norm, void *stream);
SGR_API int sgr_poisson_vcycle(int32_t depth, float *const *u, float *const *b, const float *const *q, double *partial,
                               double *norm, void *stream);
SGR_API int sgr_poisson_interpolate(int32_t N, const float *grid, int64_t m, const float *points, int32_t stride,
                                    float scale, float offset, float *values, double *partial, double *sum,
                                    void *stream);

/* ------------------------------------------------------------------------------------------
 * Quadric edge-collapse decimation (open3d's simplify_quadric_decimation with maximum_error = inf and
 * boundary_weight = 1, as coarse_mesh.py:433-463 and :716-744 call it), restated in oracle/decimate_oracle.py:
 * rounds of independent collapses until the face count is at most `target` or no edge can be collapsed.  The
 * result equals decimate_rounds of the oracle array for array.  Everything runs on `stream`; one host read per round.
 *   verts f32[V,3], faces i64[F,3] (ids in [0, V), no face repeats a vertex; checked on the device before any other
 *   work), colors / normals f32[V,3] or NULL (each goes with its output).  Outputs are caller-sized: verts_out
 *   f32[V,3], faces_out i64[F,3], colors_out / normals_out f32[V,3]; the first V' and F' rows are written: the faces
 *   that survive in their order, and the vertices they reference in theirs.
 *   result i64[4] <- V', F', rounds, faces removed by the collapse that reached the target (0 if it was not reached).
 *   Limits: V <= 2^30, F <= 2^29.  `scratch`: sgr_decimate_scratch_bytes(V, F) bytes.
 * ------------------------------------------------------------------------------------------ */
SGR_API size_t sgr_decimate_scratch_bytes(int32_t V, int32_t F);
SGR_API int sgr_decimate(int32_t V, int32_t F, int64_t target, const float *verts, const int64_t *faces,
                         const float *colors, const float *normals, float *verts_out, int64_t *faces_out,
                         float *colors_out, float *normals_out, int64_t *result, void *scratch, void *stream);

/* ------------------------------------------------------------------------------------------
 * Densification and pruning of the coarse model (SuGaRDensifier, sugar_densifier.py), restated in
 * oracle/densify_oracle.py; sugar_b200/densify.py is the caller.  P original rows, float32 raw parameters.
 * sgr_densify_stats: update_densification_stats for rows with visibility[i] != 0: max_radii = max(max_radii,
 *   float(radii)), accum += sqrtf(gx*gx + gy*gy) (each square rounded: torch's vector_norm over two floats),
 *   denom += 1.  grad_means2D f32 rows of grad_stride >= 2 floats (gx, gy first), radii i32[P], visibility u8[P],
 *   accum / denom / max_radii f32[P].  No host synchronisation.
 * sgr_densify_classify: flags u8[4,P] fully written: row 0 keep (an original row that is not split and not pruned),
 *   row 1 clone_kept, row 2 split, row 3 children_kept (both children of a split row share one fate), from accum /
 *   denom f32[P], scales (log) f32[P,3], densities (logit) f32[P] and the float32 gates below.
 * sgr_densify_emit: the P' = n_keep + n_clone + 2 n_child output rows of every column, in the order kept originals,
 *   kept clones, kept children of copy 0, kept children of copy 1 (each in parent order).  scan i32[4,P] is the
 *   inclusive scan of the four flag rows along P, and n_keep, n_clone, S, n_child its totals.  cols: a HOST array of
 *   n_cols <= SGR_DENSIFY_MAX_COLUMNS columns, src f32[P,width] -> dst f32[P',width].  Clone and child rows copy src
 *   except in SGR_DENSIFY_ZERO_NEW columns (zeros: Adam moments); a child's SGR_DENSIFY_POINTS value is
 *   R(q / |q|) (normal * exp(scale)) + point with normals f32[2S,3] (copy k of the split row of rank r reads row
 *   k*S + r; R as pytorch3d's quaternion_to_matrix) and its SGR_DENSIFY_SCALES value log(exp(scale) * inv_split).
 *   An SGR_DENSIFY_POINTS_VANILLA column is the same with R = build_rotation(q) of vanilla 3DGS
 *   (utils/general_utils.py:78-99: norm = sqrt(((r*r + x*x) + y*y) + z*z), q / norm, no epsilon, then its nine
 *   entries as written).
 *   points / scales f32[P,3] and quaternions f32[P,4] (16-byte aligned) are the parents'.  src_row i32[P'] scratch.
 *   Pruning by a mask is the same call with only the keep row set.
 * ------------------------------------------------------------------------------------------ */
#define SGR_DENSIFY_MAX_COLUMNS 24
#define SGR_DENSIFY_COPY 0      /* new rows copy the parent */
#define SGR_DENSIFY_ZERO_NEW 1  /* new rows are zero */
#define SGR_DENSIFY_POINTS 2    /* children compute their position */
#define SGR_DENSIFY_SCALES 3    /* children compute their log-scale */
#define SGR_DENSIFY_POINTS_VANILLA 4 /* SGR_DENSIFY_POINTS with vanilla 3DGS's build_rotation for R */
typedef struct SgrDensifyColumn {
    const float *src;
    float *dst;
    int32_t width;  /* floats per row */
    int32_t kind;   /* SGR_DENSIFY_* */
} SgrDensifyColumn;
/* Thresholds as float32 (torch compares a float32 tensor with a Python float rounded to float32). */
typedef struct SgrDensifyGates {
    float max_grad;     /* clone / split when the mean gradient >= max_grad */
    float clone_scale;  /* percent_dense * extent: clone when max(scale) <= it, split when > */
    float big_scale;    /* 0.1 * extent */
    float min_opacity;  /* prune when sigmoid(density) < min_opacity */
    float screen_size;  /* max_screen_size: compared with max_radii2D, all zeros after the appends */
    float inv_split;    /* 1 / (0.8 * 2) as the float reciprocal torch multiplies by */
    int32_t use_screen; /* max_screen_size is truthy: the screen and world-size clauses apply */
} SgrDensifyGates;
SGR_API int sgr_densify_stats(int32_t P, const float *grad_means2D, int32_t grad_stride, const int32_t *radii,
                              const uint8_t *visibility, float *accum, float *denom, float *max_radii, void *stream);
SGR_API int sgr_densify_classify(int32_t P, const float *accum, const float *denom, const float *scales,
                                 const float *densities, const SgrDensifyGates *gates, uint8_t *flags, void *stream);
SGR_API int sgr_densify_emit(int32_t P, int32_t n_keep, int32_t n_clone, int32_t S, int32_t n_child,
                             const int32_t *scan, int32_t n_cols, const SgrDensifyColumn *cols, const float *points,
                             const float *scales, const float *quaternions, const float *normals, float inv_split,
                             int32_t *src_row, void *stream);

/* ---- Adam step (csrc/sgr_adam.cu): the trainers' optimizer update, every parameter group in one launch -------------
 * sugar_b200/optim.py is the caller.  Each segment is one float32 parameter tensor of n elements with its gradient and
 * Adam moments, all updated in place; the scalars are torch's foreach Adam's for this step, computed on the host in
 * float64 and rounded to float32:
 *   one_minus_beta1 = 1 - beta1, beta2, one_minus_beta2 = 1 - beta2, bias_correction2_sqrt = (1 - beta2^t)^0.5,
 *   eps, step_size = -(lr / (1 - beta1^t)).
 * Per element, each op rounded on its own as torch's foreach kernels round it: m = lerp(m, g, 1 - beta1) (ATen's
 * lerp), v = v * beta2 + (1 - beta2) * (g * g), d = sqrt(v) / bias_correction2_sqrt + eps, p = p + step_size * (m / d).
 * 0 <= n <= 2^31 - 1, no null pointer in a segment with n > 0, n_segs <= SGR_ADAM_MAX_SEGMENTS; segs is a HOST
 * array.  Any float offset is legal (float4 accesses when a segment's four pointers are 16-byte aligned).  No host
 * synchronisation.
 * ------------------------------------------------------------------------------------------ */
#define SGR_ADAM_MAX_SEGMENTS 8
typedef struct SgrAdamSegment {
    float *param;
    const float *grad;
    float *exp_avg;
    float *exp_avg_sq;
    int64_t n;
    float one_minus_beta1;
    float beta2;
    float one_minus_beta2;
    float bias_correction2_sqrt;
    float eps;
    float step_size;   /* negative */
} SgrAdamSegment;
SGR_API int sgr_adam_step(int32_t n_segs, const SgrAdamSegment *segs, void *stream);

/* ------------------------------------------------------------------------------------------
 * Ground-truth image preparation (sugar_b200/dataset.py): a host-decoded image to the float32 [3,H,W] image the
 * trainers compare against, byte for byte as the reference prepares it with Pillow and numpy (PILtoTorch after
 * Image.resize, gaussian_splatting/utils/general_utils.py:21-27; the composites of dataset_readers.py:204-210 and
 * sugar_scene/cameras.py:102-107):
 *   src      u8[H_in, W_in, C]   C = 3 (RGB) or 4 (RGBA)
 *   mode     SGR_IMAGE_PLAIN        the RGB channels as they are (C = 4: only at an unchanged size, the alpha dropped)
 *            SGR_IMAGE_COMPOSITE    C = 4 over a white (white = 1) or black background in float64:
 *                                   byte = trunc((c/255 a/255 + bg (1 - a/255)) 255)
 *            SGR_IMAGE_PREMULTIPLY  C = 4 resized through premultiplied RGBa (Pillow's RGBA resize); the alpha is
 *                                   resized with the colour and then dropped
 *   x_bounds i32[W_out, 2], x_coeffs i32[W_out, kx]   Pillow's bicubic tables (xmin, count) and 22-bit fixed-point
 *   y_bounds i32[H_out, 2], y_coeffs i32[H_out, ky]   weights, as sugar_b200/dataset.py: resample_coeffs builds
 *                                   them; read only for an axis whose size changes (W_out != W_in, H_out != H_in)
 *   tmp      u8[H_in, W_out, 4]  the horizontal pass's output when both axes change (3 bytes per pixel used unless
 *                                   mode is SGR_IMAGE_PREMULTIPLY); not read otherwise and may be NULL
 *   out      f32[3, H_out, W_out]  u / 255 of each prepared byte (a correctly rounded float32 division)
 * The horizontal pass runs first, as in Pillow; each pass accumulates in int32 from 1 << 21, shifts by 22 and clamps
 * to [0, 255].  One launch per pass, none when both sizes are unchanged but a conversion pass.
 * Limits: every size >= 1, kx, ky >= 1 where their tables are read.
 * ------------------------------------------------------------------------------------------ */
#define SGR_IMAGE_PLAIN 0
#define SGR_IMAGE_COMPOSITE 1
#define SGR_IMAGE_PREMULTIPLY 2
SGR_API int sgr_image_prepare(int32_t H_in, int32_t W_in, int32_t C, int32_t mode, int32_t white, int32_t W_out,
                              int32_t kx, const int32_t *x_bounds, const int32_t *x_coeffs, int32_t H_out, int32_t ky,
                              const int32_t *y_bounds, const int32_t *y_coeffs, const uint8_t *src, uint8_t *tmp,
                              float *out, void *stream);

/* ------------------------------------------------------------------------------------------
 * LPIPS, VGG16 v0.1 (the metric of metrics.py, gaussian_splatting/lpipsPyTorch; sugar_b200/lpips.py sequences the
 * passes).  The N renders x and N ground truths y run through the network as one batch of 2N images, x first.
 * Activations are NHWC float32 [2N, H, W, C].  conv3x3 runs on the tensor cores: it rounds its input to TF32 and
 * reads its weights as TF32, so pass them rounded (to nearest, ties away: sugar_b200/lpips.py: tf32_round);
 * accumulation is float32.  conv1 is float32 throughout.
 *   weights   the packed blob, sgr_lpips_weight_floats() floats: for each of the 13 convs its weights KRSC
 *             [Cout, 3, 3, Cin] (TF32-rounded but conv1_1's) then its bias [Cout]; then the five linear vectors
 *             [64], [128], [256], [512], [512]
 *   conv1     x, y f32[N, 3, H, W] (values in [0, 1]) -> out [2N, H, W, 64]: z-score (v - mean) / std in float32,
 *             conv1_1 with zero padding of the z-scored image, bias, ReLU.  2 N H W 64 < 2^31.
 *   conv3x3   in [B, H, W, Cin] -> out [B, H, W, Cout]: 3x3 conv, stride 1, zero padding 1, bias, ReLU;
 *             Cin, Cout in {64, 128, 256, 512}; in, weight, out 16-byte aligned; B H W max(Cin, Cout) < 2^31.
 *   tap       feat [2N, H, W, C], lin f32[C], C in {64, 128, 256, 512}: per pixel of pair n (images n, N + n)
 *             sum_c lin[c] (fx_c / (|fx| + 1e-10) - fy_c / (|fy| + 1e-10))^2, summed per CTA in double into
 *             partials (N x the tap's CTA count, from sgr_lpips_scratch_layout); pooled (may be NULL) <- the 2x2 max
 *             pool [2N, H/2, W/2, C] (floored) of feat.
 *   reduce    after the five taps of an H x W input: taps f32[N, 5] (may be NULL) <- each tap's mean over its own
 *             (H >> t) x (W >> t) pixels, out f32[N] <- their sum; fixed summation order (run-to-run identical, and
 *             the same for an image whatever batch it is in).  H, W >= 16.
 * Scratch of an H x W input: sgr_lpips_scratch_layout walks its carve and writes offsets[8]: [0], [1] the two
 * activation buffers (2 N H W 64 floats each), [2 + t] tap t's partials, as byte offsets from `scratch`, and [7] the
 * bytes to allocate.  Call it with scratch = NULL for the size, then with the allocation for its offsets.
 * ------------------------------------------------------------------------------------------ */
SGR_API size_t sgr_lpips_weight_floats(void);
SGR_API int sgr_lpips_scratch_layout(int32_t N, int32_t H, int32_t W, const void *scratch, size_t *offsets);
SGR_API int sgr_lpips_conv1(int32_t N, int32_t H, int32_t W, const float *x, const float *y, const float *weight,
                            const float *bias, float *out, void *stream);
SGR_API int sgr_lpips_conv3x3(int32_t B, int32_t H, int32_t W, int32_t Cin, int32_t Cout, const float *in,
                              const float *weight, const float *bias, float *out, void *stream);
SGR_API int sgr_lpips_tap(int32_t N, int32_t H, int32_t W, int32_t C, const float *feat, const float *lin,
                          float *pooled, double *partials, void *stream);
SGR_API int sgr_lpips_reduce(int32_t N, int32_t H, int32_t W, const double *partials, float *taps, float *out,
                             void *stream);

/* Measurement hooks (bench.py): number of kernels this library has launched in this process;
 * optional CUDA-event bracketing of every launch on its own stream.  sgr_profile_read fills
 * total_ms[kind] / counts[kind] for kind < sgr_num_kernel_kinds() and resets the log. */
SGR_API unsigned long long sgr_launch_count(void);
SGR_API int sgr_num_kernel_kinds(void);
SGR_API const char *sgr_kernel_name(int kind);
SGR_API int sgr_profile_enable(int on);
SGR_API int sgr_profile_read(float *total_ms, int *counts);
SGR_API int sgr_profile_timeline(int max_records, int *kinds, float *t_begin_ms, float *t_end_ms);

/* sizeof of an ABI struct as the library was compiled (0 SgrView, 1 SgrGaussians, 2 SgrBackwardPlan, 3 SgrFieldParams,
 * 4 SgrSsimParams, 5 SgrDensifyGates, 6 SgrDensifyColumn, 7 SgrAdamSegment, 8 SgrPeerPlan; else 0): lets a foreign-language binding
 * check its own struct layout. */
SGR_API size_t sgr_struct_bytes(int32_t which);
SGR_API const char *sgr_last_error(void);
SGR_API const char *sgr_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SUGAR_B200_H_ */
