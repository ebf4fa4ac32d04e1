// sgr_backward.cu -- backward path of the H100 rasterizer.
//
// Replaces (reference: gaussian_splatting/submodules/diff-gaussian-rasterization/cuda_rasterizer/)
//   renderCUDA (backward)     backward.cu:399-557  -> blend_backward_kernel
//   computeCov2DCUDA          backward.cu:144-274  \
//   preprocessCUDA (backward) backward.cu:346-396   > preprocess_backward_kernel (one fused pass)
//   computeColorFromSH / computeCov3D backward :20-139, :278-341 /
//   9x torch::zeros           rasterize_points.cu:151-159 -> outputs fully written by the kernel;
//                              only the 48 B/Gaussian accumulator record is memset.
//
// The reference issues 9 global atomicAdd per contributing (pixel, Gaussian) pair, up to 256-way
// contended.  Here a warp parks the two per-pair scalars of its 32 pixels in shared memory, reduces 16
// splats at a time in a transposed pass and issues two 16-byte vector reductions
// (red.global.add.v4.f32 -> SASS REDG.E.ADD.F32x4) plus one scalar per (8x4 block, Gaussian): 3 L2
// operations instead of 9 per (pixel, Gaussian).
#include "sgr_internal.cuh"
#include "sgr_sh.cuh"

namespace sgr {

// Record pipeline of the backward blend: BWD_NS stages of BWD_B records with full / empty mbarriers.  A warp waits
// only for the loader warps' data, never for its sibling warps, so the tile's eight warps may drift BWD_NS - 2 batches
// apart and the statistical imbalance between the blocks of one batch is averaged over more records.
// 64-record batches in four stages (55.6 KB per CTA) rather than 96 in three (57.2 KB): the warps may drift 128
// records apart instead of 96, so fewer of them wait on a slower sibling's stage release; measured on the headline
// step (H100 SXM, 400 W): 0.98-0.99 ms against 1.01-1.02 ms, and 1.01 ms for 32 records in eight stages.
constexpr int BWD_B = 64;   // Gaussians per shared-memory batch (loader threads: the first BWD_B of the CTA)
constexpr int BWD_NS = 4;   // record stages
constexpr int BWD_NW = 8;   // warps per CTA (16x16 pixels)

// Blend accumulators (zeroed by a memset before the blend pass):
//   gacc   f32[P][8]  (dmean2D.x, dmean2D.y, dconic.x, dconic.y | dconic.w, dopacity, -, -)   in the scratch buffer
//   dcol   f32[P][3]  dL/dRGB, accumulated straight into the caller's dL_dcolors output.  With SH colours the
//          channels the forward clamped (forward.cu:63-70) are masked here, so this array IS the per-view
//          SH factor the view-parallel step exchanges, complete as soon as the blend pass ends.
__device__ __forceinline__ void red_add_v2(float *addr, float a, float b)
{
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// ------------------------------------------------------------------------------------------------
// blend backward.  One CTA per 16x16 tile, one thread per pixel, one warp per 8x4 pixel block (the
// forward's geometry); the tile's list is walked back to front over its first max(n_contrib)
// positions only, a batch of BWD_B records at a time, with the footprint masks deciding which warp
// visits which splat (sgr_internal.cuh).  Splat records move through a four-stage cp.async (LDGSTS) pipeline
// with full / empty mbarriers: the copies of batch b+1 are in flight while batch b is processed, and no warp
// ever waits for a sibling warp, only for data.
//
// Reduction.  The 9 per-pair values are NOT reduced across the warp with shuffles.  Phase 1 (lane =
// pixel) parks S = dL/dG * G and the colour weight alpha*T of every contributing splat in a per-warp
// [pixel][slot] shared-memory tile, and lane `slot` keeps the splat's batch slot in a register.  The
// splat's metadata (centre, conic, opacity, clamp bits, id) is copied out of the record stage by 16 lanes at
// once, when the chunk is flushed or before the warp releases the stage, not by every lane on every visit.
// After CH splats the warp turns around (phase 2, lane = slot x half
// block): each lane walks the 16 pixels of its half, accumulates RAW moments of S about the half's
// centre -- the pixel offsets are compile-time constants, so a pixel costs 3 FMAs for the moments and 3
// for the colours -- shifts them to the splat's centre once, combines the two halves with one xor-16
// shuffle per value and adds the result to the per-Gaussian accumulators with two red.v4 + one scalar
// reduction (chunks are ~94 % full on the headline scene).
//
// alpha is recomputed as in the forward; G = exp(power) comes from ex2.approx (MUFU.EX2) instead of
// libdevice's expf -- 2 instructions instead of 8 -- except within 1e-5 (relative) of the 1/255 threshold,
// where the exact expf decides, so the set of contributing pairs is the forward's.
// ------------------------------------------------------------------------------------------------
#ifdef SGR_BLEND_STATS
__device__ unsigned long long g_bwd_stats[8];
#define BWD_STAT(k, v) atomicAdd(&g_bwd_stats[k], (unsigned long long)(v))
int read_bwd_stats(unsigned long long *out, int reset)
{
    SGR_CUDA(cudaMemcpyFromSymbol(out, g_bwd_stats, sizeof(unsigned long long) * 8));
    if (reset) {
        unsigned long long z[8] = {};
        SGR_CUDA(cudaMemcpyToSymbol(g_bwd_stats, z, sizeof(z)));
    }
    return SGR_OK;
}
#endif
constexpr int CH = 16;             // splats per chunk
constexpr int CH_PITCH = CH + 1;   // float2 elements per pixel row: odd pitch = conflict-free transpose
// per-warp chunk scratch (bytes from its base): pair[32][CH_PITCH] float2 | meta[CH] x 32 B | dp[32] float4
//   meta: (x, y, conic a, conic b) (conic c, opacity, clamp bits, id) -- what phase 2 needs of a parked splat
//         (copied from the record stage by stash_meta)
//   dp:   (dL/dpixel r g b, -T_final <bg, dL/dpixel>) of the block's pixels
// (55.6 KB per CTA in total with four record stages of 64: four CTAs per SM fit, with 64 registers per thread; three
// CTAs with 80 registers measured 1.13 ms against 1.05 ms on the headline step, H100 SXM at 400 W, with the earlier
// three stages of 96)
constexpr uint32_t CB_META = 32 * CH_PITCH * 8, CB_DP = CB_META + CH * 32, CB_BYTES = CB_DP + 32 * 16;
// CTA shared-memory map (dynamic): the record stages, their membership words, the mbarriers, chunk scratch
constexpr uint32_t SM_A = 0, SM_B = SM_A + BWD_NS * BWD_B * 16, SM_C = SM_B + BWD_NS * BWD_B * 16,
                   SM_MEMBER = SM_C + BWD_NS * BWD_B * 16,
                   SM_BAR = SM_MEMBER + BWD_NS * BWD_NW * (BWD_B / 32) * 4,  // full[BWD_NS], empty[BWD_NS]
                   SM_LAST = SM_BAR + 2 * BWD_NS * 8, SM_CHUNK = SM_LAST + 16,
                   BWD_SMEM_BYTES = SM_CHUNK + BWD_NW * CB_BYTES;
static_assert(SM_BAR % 8 == 0 && BWD_B % 32 == 0, "mbarriers are 8-byte aligned; a batch is whole membership words");
static_assert(4 * (BWD_SMEM_BYTES + 1024) <= 228 * 1024, "four CTAs of the backward blend must fit one SM's shared memory");
// The feature blend (FEAT) adds 1 KB: the records' values, one f32 per stage slot, behind the plain layout.  Its dp
// table holds (dL/dpixel r g b, dL/dpixel feature), so phase 2 gets the fourth channel from the load it already does;
// the background term -T_final (<bg, dL/dpixel> + bg_feature dL/dpixel_feature) moves to the spare (pitch) column of
// the pixel's row of the pair tile.  The chunk scratch keeps its size, and four CTAs still fit.
constexpr uint32_t SM_V = BWD_SMEM_BYTES, BWD_SMEM_BYTES_FEAT = SM_V + BWD_NS * BWD_B * 4;
static_assert(4 * (BWD_SMEM_BYTES_FEAT + 1024) <= 228 * 1024, "four CTAs of the feature blend must fit one SM");
__host__ __device__ constexpr uint32_t CB_BGT(uint32_t px) { return (px * CH_PITCH + CH) * 8u; }

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrives on `bar` when all cp.async copies this thread has issued so far have landed (does not change the
// barrier's pending count: the expected count must include it)
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t *bar)
{
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float ex2_approx(float x)
{
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// phase 2: reduce the parked chunk (nf splats) over the block's pixels and add it to the Gaussians'
// accumulators.  Lane = (chunk slot, half): half h holds block rows 2h, 2h+1 = phase-1 lanes 16h..16h+15.
// FEAT: also c3 = sum of dchannel * dL/dpixel(feature) over the pixels, added to dval[id] (no clamp mask)
template <bool FEAT>
__device__ __forceinline__ void chunk_flush(uint32_t cb, int nf, float blk_x0, float blk_y0, float ddelx_dx,
                                            float ddely_dy, float *__restrict__ gacc, float *__restrict__ dcol,
                                            float *__restrict__ dval)
{
    const unsigned lane = threadIdx.x & 31u;
    const int slot = (int)(lane & (CH - 1)), half = (int)(lane >> 4);
    __syncwarp();
    const float4 M0 = lds128(cb + CB_META + slot * 32), M1 = lds128(cb + CB_META + slot * 32 + 16);
    const uint32_t clamp = __float_as_uint(M1.z), id = __float_as_uint(M1.w);
    // d = mean - pixel = (ax - cx_i, ay - cy_i) with the half's centre as origin: cx_i = (i & 7) - 3.5,
    // cy_i = (i >> 3) - 0.5
    const float ax = M0.x - (blk_x0 + 3.5f), ay = M0.y - (blk_y0 + 2.0f * (float)half + 0.5f);
    float s_lo = 0.f, s_hi = 0.f, t_lo = 0.f, t_hi = 0.f, u = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
    const uint32_t pa = cb + (half * 16 * CH_PITCH + slot) * 8, da = cb + CB_DP + half * 16 * 16;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const float2 pr = lds64(pa + i * CH_PITCH * 8);
        const float4 d = lds128(da + i * 16);
        const float cx = (float)(i & 7) - 3.5f;
        if (i < 8) {
            s_lo += pr.x;
            t_lo = fmaf(pr.x, cx, t_lo);
        } else {
            s_hi += pr.x;
            t_hi = fmaf(pr.x, cx, t_hi);
        }
        u = fmaf(pr.x, cx * cx, u);
        c0 = fmaf(pr.y, d.x, c0);
        c1 = fmaf(pr.y, d.y, c1);
        c2 = fmaf(pr.y, d.z, c2);
        if (FEAT) c3 = fmaf(pr.y, d.w, c3);
    }
    const float s0 = s_lo + s_hi, sx = t_lo + t_hi, sy = 0.5f * (s_hi - s_lo), sxy = 0.5f * (t_hi - t_lo);
    float m0 = s0;
    float m1 = fmaf(ax, s0, -sx);                                    // sum S dx
    float m2 = fmaf(ay, s0, -sy);                                    // sum S dy
    float m3 = fmaf(ax, fmaf(ax, s0, -2.0f * sx), u);                // sum S dx^2
    float m4 = fmaf(ax, m2, fmaf(-ay, sx, sxy));                     // sum S dx dy
    float m5 = fmaf(ay, fmaf(ay, s0, -2.0f * sy), 0.25f * s0);       // sum S dy^2
    m0 += __shfl_xor_sync(0xffffffffu, m0, 16);
    m1 += __shfl_xor_sync(0xffffffffu, m1, 16);
    m2 += __shfl_xor_sync(0xffffffffu, m2, 16);
    m3 += __shfl_xor_sync(0xffffffffu, m3, 16);
    m4 += __shfl_xor_sync(0xffffffffu, m4, 16);
    m5 += __shfl_xor_sync(0xffffffffu, m5, 16);
    c0 += __shfl_xor_sync(0xffffffffu, c0, 16);
    c1 += __shfl_xor_sync(0xffffffffu, c1, 16);
    c2 += __shfl_xor_sync(0xffffffffu, c2, 16);
    if (FEAT) c3 += __shfl_xor_sync(0xffffffffu, c3, 16);
    if (slot < nf) {
        // moments -> gradients (backward.cu:537-554): dG/ddel = -G (Q d)
        float *g = gacc + (size_t)id * 8, *dc = dcol + (size_t)id * 3;
        if (half == 0) {
            const float gmx = -(M0.z * m1 + M0.w * m2) * ddelx_dx;
            const float gmy = -(M1.x * m2 + M0.w * m1) * ddely_dy;
            red_add_v4(g, gmx, gmy, -0.5f * m3, -0.5f * m4);
            if (!(clamp & 1u)) atomicAdd(dc, c0);
            if (FEAT) atomicAdd(dval + id, c3);
        } else {
            red_add_v2(g + 4, -0.5f * m5, __fdividef(m0, M1.y));
            if (!(clamp & 2u)) atomicAdd(dc + 1, c1);
            if (!(clamp & 4u)) atomicAdd(dc + 2, c2);
        }
    }
    __syncwarp();
}

// FEAT: the feature channel of the forward's FEAT blend: values[P], its background *feat_bg, dL/d(feature map)
// dL_dfeat[H,W] in, dL/dvalues into dval[P]; the FEAT = false instantiations ignore the last four arguments.
template <bool packed, bool FEAT>
__global__ void __launch_bounds__(256, 4) blend_backward_kernel(
    const uint32_t *__restrict__ tile_order, const uint32_t *__restrict__ tile_start, const uint32_t *__restrict__ tile_end,
    const uint32_t *__restrict__ plist, const float4 *__restrict__ rec, int W, int H, int gx, const float *__restrict__ bg,
    const float *__restrict__ final_Ts, const uint32_t *__restrict__ n_contrib, const float *__restrict__ dL_dpixels,
    float *__restrict__ gacc, float *__restrict__ dcol, const float *__restrict__ values,
    const float *__restrict__ feat_bg, const float *__restrict__ dL_dfeat, float *__restrict__ dval)
{
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int tile = (int)tile_order[blockIdx.x];
    // the forward's live list of the tile; n_contrib counts positions in it
    const uint32_t lo = tile_start[tile], hi = tile_end[tile];
    if (hi == lo) return;
    const int tile_y = tile / gx, tile_x = tile - tile_y * gx;
    const int tid = threadIdx.x;
    const unsigned lane = tid & 31, wid = tid >> 5;
    const int tx0 = tile_x * SGR_TILE, ty0 = tile_y * SGR_TILE;
    const int bx0 = tx0 + (int)(wid & 1u) * 8, by0 = ty0 + (int)(wid >> 1) * 4;
    const uint32_t pxi = bx0 + (lane & 7u), pyi = by0 + (lane >> 3);
    const bool inside = pxi < (uint32_t)W && pyi < (uint32_t)H;
    const uint32_t sm = smem_addr_pinned(s_raw);
    int *s_tile_last = (int *)(s_raw + SM_LAST);
    uint32_t(*s_member)[BWD_B / 32] = (uint32_t(*)[BWD_B / 32])(s_raw + SM_MEMBER);
    if (tid == 0) *s_tile_last = 0;

    const size_t pix = (size_t)pyi * W + pxi, plane = (size_t)H * W;
    float T = inside ? final_Ts[pix] : 0.0f;
    const int last_contributor = inside ? (int)n_contrib[pix] : 0;
    const uint32_t cb = sm + SM_CHUNK + wid * CB_BYTES;
    {
        float dp0 = 0.f, dp1 = 0.f, dp2 = 0.f, dp3 = 0.f;
        if (inside) {
            dp0 = dL_dpixels[pix];
            dp1 = dL_dpixels[plane + pix];
            dp2 = dL_dpixels[2 * plane + pix];
            if (FEAT) dp3 = dL_dfeat[pix];
        }
        // (dL/dpixel, -T_final * <bg, dL/dpixel>) of this pixel: phase 2 reads the block's table; the
        // hit path of phase 1 reloads its own entry instead of pinning four registers across the loop
        const float bgdp = fmaf(bg[2], dp2, fmaf(bg[1], dp1, bg[0] * dp0));
        if (FEAT) {  // (dL/dpixel r g b feature) in the table, the background term in the pair tile's spare column
            sts128(cb + CB_DP + lane * 16, dp0, dp1, dp2, dp3);
            sts32(cb + CB_BGT(lane), __float_as_uint(-T * fmaf(feat_bg[0], dp3, bgdp)));
        } else {
            sts128(cb + CB_DP + lane * 16, dp0, dp1, dp2, -T * bgdp);
        }
    }
    // the pixel centre, pinned: under register pressure nvcc otherwise re-derives it from special
    // registers inside the splat loop
    float pxf = (float)pxi, pyf = (float)pyi;
    asm volatile("mov.f32 %0, %0;" : "+f"(pxf));
    asm volatile("mov.f32 %0, %0;" : "+f"(pyf));
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    // Splats behind the deepest last contributor of the warp (of the tile) cannot touch any of its
    // pixels: the tile only walks list positions [0, tile_last), each warp only [0, warp_last).
    const int warp_last = __reduce_max_sync(0xffffffffu, last_contributor);
    __syncthreads();
    if (lane == 0 && warp_last > 0) atomicMax(s_tile_last, warp_last);
    __syncthreads();
    const int n = *s_tile_last;
    if (n == 0) return;
    int nfill = 0;
    const float blk_x0 = (float)bx0, blk_y0 = (float)by0;

    // record pipeline (threads 0..BWD_B-1 own one slot of every batch)
    const bool loader = tid < BWD_B;
    auto fetch = [&](int b0) -> uint32_t {
        // back to front; 0xffffffff: no slot (the live list holds no dead instance: scatter left them out)
        if (!(loader && b0 + tid < n)) return 0xffffffffu;
        return plist[lo + (uint32_t)(n - 1 - (b0 + tid))];
    };
    // membership words of the batch in stage `st` from the loader threads' masks
    auto publish_members = [&](uint32_t mask, uint32_t(*set)[BWD_B / 32]) {
#pragma unroll
        for (int blk = 0; blk < BWD_NW; blk++) {
            const uint32_t word = __ballot_sync(0xffffffffu, (mask >> blk) & 1u);
            if (lane == 0) set[blk][wid] = word;
        }
    };
    uint64_t *bars = (uint64_t *)(s_raw + SM_BAR);  // full[0..BWD_NS) then empty[0..BWD_NS)
    if (tid == 0) {
        for (int st = 0; st < BWD_NS; st++) {
            mbar_init(&bars[st], 2 * BWD_B);         // per loader thread: one async arrive (copies landed) + one plain
            mbar_init(&bars[BWD_NS + st], BWD_NW);  // one arrive per warp when it is done with the stage
        }
        mbar_fence_init();
    }
    __syncthreads();
    const int nb = (n + BWD_B - 1) / BWD_B;
    // loader warps: fill stage b % BWD_NS with batch b (waits until every warp has released the stage's previous batch)
    auto produce = [&](int b) {
        const int st = b % BWD_NS;
        if (b >= BWD_NS) mbar_wait(&bars[BWD_NS + st], (uint32_t)((b / BWD_NS - 1) & 1));
        const uint32_t w = fetch(b * BWD_B);
        uint32_t mask = 0;
        if (w != 0xffffffffu) {
            const uint32_t id = packed ? (w >> 8) : w;
            const float4 *r = rec + (size_t)id * 3;
            const uint32_t e = st * BWD_B + tid;
            cp_async16_a(sm + SM_A + e * 16, r);
            cp_async16_a(sm + SM_B + e * 16, r + 1);
            cp_async16_a(sm + SM_C + e * 16, r + 2);
            if (FEAT) cp_async4_a(sm + SM_V + e * 4, values + id);
            if (packed) mask = w & 0xffu;
        }
        if (!packed) {  // the mask needs the landed record
            cp_async_commit();
            cp_async_wait<0>();
            if (w != 0xffffffffu) {
                const float4 r0 = lds128(sm + SM_A + (st * BWD_B + tid) * 16), r1 = lds128(sm + SM_B + (st * BWD_B + tid) * 16);
                mask = block_mask_of_record(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, tx0, ty0);
            }
        }
        cp_async_mbar_arrive_noinc(&bars[st]);
        publish_members(mask, s_member + st * BWD_NW);
        mbar_arrive(&bars[st]);
    };
    // Chunk slots [0, nfill) hold parked pairs; the metadata of slots [0, nmeta) is already in the chunk's meta rows.
    // A slot parked from the current stage only records its batch slot (lane `slot`'s pj); its metadata is copied
    // out of the stage by stash_meta, once per flush and once before the stage is released.
    int nmeta = 0, pj = 0;
    auto stash_meta = [&](uint32_t sa, uint32_t sb, uint32_t sc, int to) {
        if ((int)lane >= nmeta && (int)lane < to) {
            const float4 A = lds128(sa + pj * 16), B = lds128(sb + pj * 16);
            const float2 Cm = lds64(sc + pj * 16 + 8);  // (clamp bits, id)
            const uint32_t ma = cb + CB_META + lane * 32;
            sts128(ma, A.x, A.y, A.z, A.w);
            sts128(ma + 16, B.x, B.z, Cm.x, Cm.y);
        }
        nmeta = to;
    };
    if (loader) produce(0);
    for (int b = 0; b < nb; b++) {
        const int b0 = b * BWD_B, buf = b % BWD_NS;
        const uint32_t sa = sm + SM_A + buf * (BWD_B * 16), sb = sm + SM_B + buf * (BWD_B * 16),
                       sc = sm + SM_C + buf * (BWD_B * 16);
        if (loader && b + 1 < nb) produce(b + 1);
        mbar_wait(&bars[buf], (uint32_t)((b / BWD_NS) & 1));  // batch b has landed and its membership words are visible
        const uint32_t(*member)[BWD_B / 32] = s_member + buf * BWD_NW;
        const int m = min(BWD_B, n - b0);
#ifdef SGR_BLEND_STATS
        if (tid == 0) BWD_STAT(6, m);
#endif
        const int jmin = n - b0 - warp_last;  // first batch slot whose list position is < warp_last
        // list position of slot j is n-1-(b0+j); it precedes this pixel's last contributor iff j > jlim
        const int jlim = n - 1 - b0 - last_contributor;
#pragma unroll 1
        for (int c = 0; c * 32 < m; c++) {
            uint32_t mw = member[wid][c];
            const int cut = jmin - c * 32;
            if (cut >= 32) mw = 0;
            else if (cut > 0) mw &= ~((1u << cut) - 1u);
#pragma unroll 1
            while (mw) {
                const int j = c * 32 + (__ffs(mw) - 1);
                mw &= mw - 1;
                const float4 A = lds128(sa + j * 16);
                const float4 B = lds128(sb + j * 16);
                const float dx = __fsub_rn(A.x, pxf), dy = __fsub_rn(A.y, pyf);
                const float power = splat_power(dx, dy, A.z, A.w, B.x);
                const bool valid = j > jlim && !(power > 0.0f) && !(power < B.y);
#ifdef SGR_BLEND_STATS
                {
                    const bool hit = valid && !(fminf(0.99f, __fmul_rn(B.z, expf(power))) < 1.0f / 255.0f);
                    const unsigned mc = __ballot_sync(0xffffffffu, valid), mh = __ballot_sync(0xffffffffu, hit);
                    const unsigned ml = __ballot_sync(0xffffffffu, j > jlim);
                    if (lane == 0) {
                        BWD_STAT(0, 1);
                        BWD_STAT(1, mc != 0);
                        BWD_STAT(2, mh != 0);
                        BWD_STAT(3, __popc(mc));
                        BWD_STAT(4, __popc(mh));
                        BWD_STAT(5, __popc(ml));
                    }
                }
#endif
                if (!__any_sync(0xffffffffu, valid)) continue;
                // S = dL/dG * G and the colour weight alpha*T of this pair; zero for lanes without one.
                // (A candidate warp almost always keeps a contributing lane, so there is no second vote:
                // an all-zero slot is harmless.)  Every lane evaluates the pair and only a contributing lane keeps
                // it: the warp issues these instructions anyway, and without the two divergent branches it saves
                // their convergence barriers.
                float G = ex2_approx(power * 1.4426950408889634f);
                float alpha = fminf(0.99f, B.z * G);
                if (valid && fabsf(alpha - 1.0f / 255.0f) < 4.0e-8f) {  // on the threshold: decide as the forward did
                    G = expf(power);
                    alpha = fminf(0.99f, __fmul_rn(B.z, G));
                }
                const bool hit = valid && !(alpha < 1.0f / 255.0f);
                const float2 Cc = lds64(sc + j * 16);
                const float4 dp = lds128(cb + CB_DP + lane * 16);
                const float om = 1.0f - alpha;  // in [0.01, 1) where kept: a bare MUFU.RCP suffices
                float inv;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(om));
                const float Tn = T * inv;
                // acc holds the colour blended behind this splat (backward.cu:493-499 keeps last_alpha /
                // last_color and folds them in one iteration later; same operations on the same values,
                // evaluated eagerly below)
                float dL_dalpha = (B.w - acc0) * dp.x;
                dL_dalpha = fmaf(Cc.x - acc1, dp.y, dL_dalpha);
                dL_dalpha = fmaf(Cc.y - acc2, dp.z, dL_dalpha);
                float fv = 0.f, bgt = dp.w;
                if (FEAT) {
                    fv = __uint_as_float(lds32(sm + SM_V + (buf * BWD_B + j) * 4));
                    dL_dalpha = fmaf(fv - acc3, dp.w, dL_dalpha);
                    bgt = __uint_as_float(lds32(cb + CB_BGT(lane)));
                }
                dL_dalpha *= Tn;
                dL_dalpha = fmaf(bgt, inv, dL_dalpha);
                const float S = hit ? B.z * dL_dalpha * G : 0.f;
                const float dchannel = hit ? alpha * Tn : 0.f;
                if (hit) {
                    acc0 = fmaf(alpha, B.w, om * acc0);
                    acc1 = fmaf(alpha, Cc.x, om * acc1);
                    acc2 = fmaf(alpha, Cc.y, om * acc2);
                    if (FEAT) acc3 = fmaf(alpha, fv, om * acc3);
                    T = Tn;
                }
                // park: every lane its pair, lane `nfill` the batch slot (the metadata follows in stash_meta)
                sts64(cb + (lane * CH_PITCH + nfill) * 8, S, dchannel);
                if ((int)lane == nfill) pj = j;
                if (++nfill == CH) {
                    stash_meta(sa, sb, sc, CH);
                    chunk_flush<FEAT>(cb, CH, blk_x0, blk_y0, 0.5f * W, 0.5f * H, gacc, dcol, dval);
                    nfill = nmeta = 0;
                }
            }
        }
        stash_meta(sa, sb, sc, nfill);  // the parked slots' metadata leaves the stage before it is released
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars[BWD_NS + buf]);  // this warp no longer reads the stage
    }
    if (nfill) chunk_flush<FEAT>(cb, nfill, blk_x0, blk_y0, 0.5f * W, 0.5f * H, gacc, dcol, dval);
}

// ------------------------------------------------------------------------------------------------
// per-Gaussian backward (cov2D inverse, projection, SH, scale/rotation), one fused pass.
// HBM-bound: every input array is staged into shared memory by 1-D bulk copies through the TMA
// engine, each thread works on its own Gaussian out of shared memory, and all outputs leave through
// coalesced stores.  The SH coefficients are not an input: the view-direction term of dL/dmean3D
// comes from the forward's Jacobian rows (36 B per Gaussian instead of the 192 B row), and the SH
// gradient is built in a shared-memory row block on its way out.
// ------------------------------------------------------------------------------------------------
struct PreBwdArgs {
    int p0, p1;  // Gaussian range of this launch (one chunk of the per-Gaussian pass); p0 % PB_T == 0
    // shs / sh_rest: only whether SH colours are present (their contents are never read)
    const float *means, *scales, *rots, *shs, *cov_pre;
    const float *sh_jac;  // [P][9] the forward's dRGB/d(dir) rows (GeomState::sh_jac)
    ViewConsts v;
    const int32_t *radii;
    const float *gacc;  // [P][8] blend accumulators
    const float *dcol;  // [P][3] accumulated dL/dRGB (= the dL_dcolors output; clamp-masked with SH)
    float *dmeans2D, *dopacity, *dmeans3D, *dcov3D, *dsh, *dscales, *drots;
    // optional f32[P][11]: (dL_dmeans3D 3 | dL_dopacity 1 | dL_dscales 3 | dL_drotations 4) of a Gaussian as ONE
    // 44-byte record instead of the four arrays (the view-parallel step all-reduces these records chunk by chunk)
    float *rec11;
    int in_bulk_ok, out_bulk_ok, sh_stride, sh_vec;
    // raw-parameter mode (SgrGaussians.activations): scales / rots are the model's raw parameters; dopacity / dscales /
    // drots / dsh / dsh_rest are gradients of the RAW parameters, dsh of the DC array and dsh_rest of the others
    const float4 *rec;  // splat records of the forward: rec[3i+1].z = the activated opacity
    float *dsh_rest;
    // view-parallel peer mode (csrc/sgr_peer.cu): dsh rows leave as the sum over ALL views' SH gradients.  view_tab is a
    // device table of nviews pointers to the views' factor blocks (f32[3P] dL/dRGB + the view's camera position at
    // campos_off), entries of other ranks pointing into THEIR memory over NVLink; view my_view is this launch's own
    // (its factor is `dcol`).  dsh_scale multiplies every dsh row (1/num_views for a mean over the batch).
    const float *const *view_tab;
    int nviews, my_view;
    size_t campos_off;
    float dsh_scale;
    // peer mode, records: CTA b of this launch (a chunk of the pass) stores its 64 records into the staging array of the
    // rank that OWNS them -- owner = b * nviews / gridDim.x, stage_tab[owner] = that rank's array for records coming
    // from this rank -- with one TMA bulk store (a posted write over NVLink): the reduce-scatter half of the records'
    // all-reduce is fused into this kernel's write-out.  NULL: records go to rec11.
    float *const *stage_tab;
    int pf_off;  // floats: where the other views' factor blocks land in shared memory (MULTI)
};

// dL/dsh of one view (backward.cu:20-139: dL/dsh_k = basis_k(dir) dL/dRGB) into one shared-memory row [M][3].
// Write-only: the view-direction term, the only use the reference makes of the coefficients, comes from the
// forward's Jacobian rows (sh_dir_grad).  `dc` is coefficient 0's row of three, `rest` coefficient 1's (one combined
// row: rest = dc + 3; raw-parameter mode: two arrays).  OTHERS: the other views' SH gradients of this Gaussian
// (registers, `oacc`) join the row here.
template <bool OTHERS = false>
__device__ __forceinline__ void sh_grad_row(int deg, int M, float *dc, float *rest, f3 d, f3 dRGB,
                                            float out_scale = 1.0f, const float *oacc = nullptr)
{
    const f3 dS = {dRGB.x * out_scale, dRGB.y * out_scale, dRGB.z * out_scale};  // x 1.0f is exact
    sh_for_active(deg, [&](auto k) {
        constexpr int K = decltype(k)::value;
        float *q = K == 0 ? dc : rest + (K - 1) * 3;
        const float w = sh_basis<K>(d);
        if constexpr (OTHERS) {
            q[0] = fmaf(w, dS.x, oacc[K * 3]);
            q[1] = fmaf(w, dS.y, oacc[K * 3 + 1]);
            q[2] = fmaf(w, dS.z, oacc[K * 3 + 2]);
        } else {
            q[0] = w * dS.x;
            q[1] = w * dS.y;
            q[2] = w * dS.z;
        }
    });
    // rows above the active degree stay zero (the reference returns zero-filled dL_dsh)
    for (int k = (deg + 1) * (deg + 1) * 3 - 3; k < (M - 1) * 3; k++) rest[k] = 0.f;
}

constexpr int PB_VB = 7;  // other views whose factors a thread fetches at the top of the kernel (8 ranks: all of them)
static_assert(PB_T == 64, "the peer record exchange (sgr_peer.cu) works in blocks of 64 records");
// dynamic shared memory carve-up (floats): inputs, outputs, then the SH block
constexpr int PB_GACC = 0;                     // PB_T*8
constexpr int PB_DCOL = PB_GACC + PB_T * 8;    // PB_T*3
constexpr int PB_MEANS = PB_DCOL + PB_T * 3;   // PB_T*3
constexpr int PB_SCALES = PB_MEANS + PB_T * 3;
constexpr int PB_ROTS = PB_SCALES + PB_T * 3;  // PB_T*4 (16B aligned: offset is a multiple of 4 floats)
constexpr int PB_COV = PB_ROTS + PB_T * 4;     // PB_T*6
constexpr int PB_O_M2D = PB_COV + PB_T * 6;    // outputs
constexpr int PB_O_COV = PB_O_M2D + PB_T * 3;
// the 11 all-reduce-bound floats per Gaussian: four arrays (OPA | M3D | SCL | ROT) or PB_T records of 11
constexpr int PB_O_R11 = PB_O_COV + PB_T * 6;
constexpr int PB_O_OPA = PB_O_R11;
constexpr int PB_O_M3D = PB_O_OPA + PB_T;
constexpr int PB_O_SCL = PB_O_M3D + PB_T * 3;
constexpr int PB_O_ROT = PB_O_SCL + PB_T * 3;  // multiple of 4 floats
constexpr int PB_SHDC = PB_O_R11 + PB_T * 11;  // raw mode: the gradient of the DC coefficients, PB_T*3
// the SH block, PB_T rows of sh_stride floats (raw mode: of 3(M-1)) and at least PB_T*9: it first receives the CTA's
// Jacobian rows (PB_T*9, read into registers before the first dL/dsh row is written), then the dL/dsh rows
constexpr int PB_SH = PB_SHDC + PB_T * 3 + (PB_T & 3 ? 4 - (PB_T & 3) : 0);
static_assert(PB_T % 4 == 0, "every region starts on a 16-byte boundary");
static_assert(PB_ROTS % 4 == 0 && PB_O_ROT % 4 == 0 && PB_SH % 4 == 0, "16-byte alignment of float4 regions");

// 1-D bulk async copy shared -> global (TMA store, no tensor map); bytes % 16 == 0, both sides 16-byte aligned
__device__ __forceinline__ void bulk_s2g(void *dst, const void *src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src_smem)),
                 "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void pb_stage(float *dst, const float *__restrict__ src, int n)
{
    for (int i = threadIdx.x; i < n; i += PB_T) dst[i] = __ldg(src + i);
}
__device__ __forceinline__ void pb_flush(float *__restrict__ dst, const float *src, int n)
{
    for (int i = threadIdx.x; i < n; i += PB_T) dst[i] = src[i];
}

// MULTI (view-parallel peer mode, never with RAW): dsh rows leave as the sum over all views, see PreBwdArgs::view_tab
template <bool RAW, bool MULTI = false>
__global__ void __launch_bounds__(PB_T) preprocess_backward_kernel(const PreBwdArgs a)
{
    extern __shared__ __align__(16) float sm[];
    __shared__ __align__(8) uint64_t s_bar;
    const int tid = threadIdx.x;
    const int base = a.p0 + blockIdx.x * PB_T;
    const int n = min(PB_T, a.p1 - base);
    const int i = base + tid;
    const int M = a.v.M;
    const bool full = (n == PB_T);

    if (a.in_bulk_ok && full) {
        if (tid == 0) {
            mbar_init(&s_bar, 1);
            mbar_fence_init();
            uint32_t bytes = PB_T * 32 + PB_T * 12;
            if (a.shs) bytes += PB_T * 12 + PB_T * 36;  // dL/dRGB and the Jacobian rows: inputs of the SH backward only
            if (a.scales) bytes += PB_T * 12 + PB_T * 16;
            if (a.cov_pre) bytes += PB_T * 24;
            // peer mode: the other views' factor blocks of these 64 Gaussians, one bulk copy per view straight out of
            // its owner GPU's memory (TMA over NVLink): the factors' all-gather is fused into this kernel's staging.
            // One barrier for everything: a separate, later-waited barrier for the pulled blocks adds a second wait
            // to every CTA of a latency-bound pass.
            const int pulled = MULTI ? min(a.nviews - 1, PB_VB) : 0;
            bytes += (uint32_t)pulled * PB_T * 12;
            mbar_expect_tx(&s_bar, bytes);
            for (int u = 0; u < pulled; u++) {
                const int v = u + (u >= a.my_view ? 1 : 0);
                bulk_g2s(sm + a.pf_off + u * PB_T * 3, a.view_tab[v] + (size_t)base * 3, PB_T * 12, &s_bar);
            }
            bulk_g2s(sm + PB_GACC, a.gacc + (size_t)base * 8, PB_T * 32, &s_bar);
            if (a.shs) {
                bulk_g2s(sm + PB_DCOL, a.dcol + (size_t)base * 3, PB_T * 12, &s_bar);
                bulk_g2s(sm + PB_SH, a.sh_jac + (size_t)base * 9, PB_T * 36, &s_bar);
            }
            bulk_g2s(sm + PB_MEANS, a.means + (size_t)base * 3, PB_T * 12, &s_bar);
            if (a.scales) {
                bulk_g2s(sm + PB_SCALES, a.scales + (size_t)base * 3, PB_T * 12, &s_bar);
                bulk_g2s(sm + PB_ROTS, a.rots + (size_t)base * 4, PB_T * 16, &s_bar);
            }
            if (a.cov_pre) bulk_g2s(sm + PB_COV, a.cov_pre + (size_t)base * 6, PB_T * 24, &s_bar);
        }
    } else {
        pb_stage(sm + PB_GACC, a.gacc + (size_t)base * 8, n * 8);
        if (a.shs) {
            pb_stage(sm + PB_DCOL, a.dcol + (size_t)base * 3, n * 3);
            pb_stage(sm + PB_SH, a.sh_jac + (size_t)base * 9, n * 9);
        }
        pb_stage(sm + PB_MEANS, a.means + (size_t)base * 3, n * 3);
        if (a.scales) {
            pb_stage(sm + PB_SCALES, a.scales + (size_t)base * 3, n * 3);
            pb_stage(sm + PB_ROTS, a.rots + (size_t)base * 4, n * 4);
        }
        if (a.cov_pre) pb_stage(sm + PB_COV, a.cov_pre + (size_t)base * 6, n * 6);
        if (MULTI) {
            const int pulled = min(a.nviews - 1, PB_VB);
            for (int u = 0; u < pulled; u++) {
                const int v = u + (u >= a.my_view ? 1 : 0);
                pb_stage(sm + a.pf_off + u * PB_T * 3, a.view_tab[v] + (size_t)base * 3, n * 3);
            }
        }
    }
    float *s_sh = sm + PB_SH;
    const int row_f = RAW ? (M - 1) * 3 : M * 3;  // floats per row of the SH block in shared memory
    int radius = 0;
    if (tid < n) radius = a.radii[i];
    const int others = MULTI ? a.nviews - 1 : 0;
    __syncthreads();
    if (a.in_bulk_ok && full) mbar_wait(&s_bar, 0);
    // dL/ddir from this Gaussian's Jacobian row, before the SH block is reused for the dL/dsh rows
    f3 ddir = {0.f, 0.f, 0.f};
    if (a.shs) {
        if (tid < n && radius > 0) {
            const f3 dRGB = {sm[PB_DCOL + tid * 3], sm[PB_DCOL + tid * 3 + 1], sm[PB_DCOL + tid * 3 + 2]};
            ddir = sh_dir_grad(s_sh + tid * 9, dRGB);  // stride 9: conflict-free
        }
        __syncthreads();
    }

    // peer mode: the other views' SH gradients of this Gaussian, summed in registers (48 accumulators); they join the
    // row when this view's gradient is written into it (or make up the whole row if the Gaussian is culled here)
    float oacc[MULTI ? 48 : 1];
    auto sum_other_views = [&]() {
        if (!MULTI) return;
#pragma unroll
        for (int k = 0; k < (MULTI ? 48 : 1); k++) oacc[k] = 0.f;
        if (others <= 0) return;
        const float mx = sm[PB_MEANS + tid * 3], my = sm[PB_MEANS + tid * 3 + 1], mz = sm[PB_MEANS + tid * 3 + 2];
        for (int u0 = 0; u0 < others; u0 += PB_VB) {
            float pf[PB_VB][3];
#pragma unroll
            for (int u = 0; u < PB_VB; u++) {
                const int uu = u0 + u, v = uu + (uu >= a.my_view ? 1 : 0);
                const bool on = uu < others;
                if (u0 == 0) {  // staged in shared memory by the bulk copies above
                    const float *g = sm + a.pf_off + u * PB_T * 3 + tid * 3;
                    pf[u][0] = on ? g[0] : 0.f;
                    pf[u][1] = on ? g[1] : 0.f;
                    pf[u][2] = on ? g[2] : 0.f;
                } else {        // more than PB_VB + 1 views: the rest straight from global / peer memory
                    const float *g = a.view_tab[on ? v : a.my_view] + (size_t)i * 3;
                    pf[u][0] = on ? __ldcg(g) : 0.f;
                    pf[u][1] = on ? __ldcg(g + 1) : 0.f;
                    pf[u][2] = on ? __ldcg(g + 2) : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < PB_VB; u++) {
                const f3 g = {pf[u][0] * a.dsh_scale, pf[u][1] * a.dsh_scale, pf[u][2] * a.dsh_scale};
                if (g.x == 0.f && g.y == 0.f && g.z == 0.f) continue;  // not visible in that view (or past the last view)
                const int uu = u0 + u, v = uu + (uu >= a.my_view ? 1 : 0);
                const float *cp = a.view_tab[v] + a.campos_off;
                sh_accumulate(a.v.D, oacc, sh_dir(mx, my, mz, __ldg(cp), __ldg(cp + 1), __ldg(cp + 2)), g);
            }
        }
    };
    if (MULTI && tid < n) sum_other_views();
    if (tid < n) {
        const bool vis = radius > 0;
        // the 11 all-reduce-bound outputs: four arrays, or one 44-byte record per Gaussian (stride 11: conflict-free)
        const bool aos = a.rec11 != nullptr;
        float *o_m2d = sm + PB_O_M2D + tid * 3, *o_cov = sm + PB_O_COV + tid * 6;
        float *o_m3d = aos ? sm + PB_O_R11 + tid * 11 : sm + PB_O_M3D + tid * 3;
        float *o_opa = aos ? o_m3d + 3 : sm + PB_O_OPA + tid;
        float *o_scl = aos ? o_m3d + 4 : sm + PB_O_SCL + tid * 3;
        float *o_rot = aos ? o_m3d + 7 : sm + PB_O_ROT + tid * 4;
        float *row = s_sh + tid * (RAW ? row_f : a.sh_stride);
        if (!vis) {
            o_m2d[0] = o_m2d[1] = o_m2d[2] = 0.f;
            *o_opa = 0.f;
            o_m3d[0] = o_m3d[1] = o_m3d[2] = 0.f;
#pragma unroll
            for (int k = 0; k < 6; k++) o_cov[k] = 0.f;
            o_scl[0] = o_scl[1] = o_scl[2] = 0.f;
            o_rot[0] = o_rot[1] = o_rot[2] = o_rot[3] = 0.f;
            if (a.shs && a.dsh) {
                if (MULTI) {
#pragma unroll
                    for (int k = 0; k < 48; k++)
                        if (k < row_f) row[k] = oacc[k];
                    for (int k = 48; k < row_f; k++) row[k] = 0.f;
                } else {
                    for (int k = 0; k < row_f; k++) row[k] = 0.f;
                }
                if (RAW) sm[PB_SHDC + tid * 3] = sm[PB_SHDC + tid * 3 + 1] = sm[PB_SHDC + tid * 3 + 2] = 0.f;
            }
        } else {
            const float4 *gr = (const float4 *)(sm + PB_GACC) + tid * 2;
            const float4 g0 = gr[0], g1 = gr[1];
            const float dmx = g0.x, dmy = g0.y;
            const float dcx = g0.z, dcy = g0.w, dcz = g1.x;
            o_m2d[0] = dmx;
            o_m2d[1] = dmy;
            o_m2d[2] = 0.f;
            // raw mode: d sigmoid = o (1 - o), with the activated opacity the forward stored in the splat record
            float act_o = 1.0f;
            if (RAW) {
                const float o = __ldg(&a.rec[(size_t)i * 3 + 1]).z;
                act_o = o * (1.0f - o);
            }
            *o_opa = g1.y * act_o;

            const float *vm = a.v.viewmatrix, *proj = a.v.projmatrix;
            const float mx = sm[PB_MEANS + tid * 3], my = sm[PB_MEANS + tid * 3 + 1], mz = sm[PB_MEANS + tid * 3 + 2];
            float c3[6];
            float4 q = make_float4(1, 0, 0, 0);
            float sc0 = 0, sc1 = 0, sc2 = 0, q_len = 1.0f;
            if (a.cov_pre) {
#pragma unroll
                for (int k = 0; k < 6; k++) c3[k] = sm[PB_COV + tid * 6 + k];
            } else {
                sc0 = sm[PB_SCALES + tid * 3], sc1 = sm[PB_SCALES + tid * 3 + 1], sc2 = sm[PB_SCALES + tid * 3 + 2];
                q = ((const float4 *)(sm + PB_ROTS))[tid];
                if (RAW) {  // the forward's activations, recomputed (sugar_model.py:417, 479)
                    sc0 = expf(sc0), sc1 = expf(sc1), sc2 = expf(sc2);
                    q_len = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
                    const float inv = __fdiv_rn(1.0f, q_len);
                    q = make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
                }
                cov3d_from_scale_rot(sc0, sc1, sc2, a.v.scale_modifier, q, c3);
            }
            // ---- computeCov2DCUDA (backward.cu:144-274) ----
            float tx = xf_row(vm, 0, mx, my, mz), ty = xf_row(vm, 1, mx, my, mz);
            const float tzv = xf_row(vm, 2, mx, my, mz);
            const float h_x = a.v.focal_x, h_y = a.v.focal_y;
            const float limx = 1.3f * a.v.tanfovx, limy = 1.3f * a.v.tanfovy;
            const float txtz = tx / tzv, tytz = ty / tzv;
            tx = fminf(limx, fmaxf(-limx, txtz)) * tzv;
            ty = fminf(limy, fmaxf(-limy, tytz)) * tzv;
            const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
            const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
            const float J00 = h_x / tzv, J02 = -(h_x * tx) / (tzv * tzv), J11 = h_y / tzv, J12 = -(h_y * ty) / (tzv * tzv);
            float T0[3], T1[3];
#pragma unroll
            for (int r = 0; r < 3; r++) {
                T0[r] = vm[4 * r] * J00 + vm[2 + 4 * r] * J02;
                T1[r] = vm[1 + 4 * r] * J11 + vm[2 + 4 * r] * J12;
            }
            const float V[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
            float p[3], qv[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                p[k] = T0[0] * V[k][0] + T0[1] * V[k][1] + T0[2] * V[k][2];
                qv[k] = T1[0] * V[k][0] + T1[1] * V[k][1] + T1[2] * V[k][2];
            }
            const float ca = T0[0] * p[0] + T0[1] * p[1] + T0[2] * p[2] + 0.3f;
            const float cb = T0[0] * qv[0] + T0[1] * qv[1] + T0[2] * qv[2];
            const float cc = T1[0] * qv[0] + T1[1] * qv[1] + T1[2] * qv[2] + 0.3f;
            const float denom = ca * cc - cb * cb;
            float dL_da = 0, dL_db = 0, dL_dc = 0;
            const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
            float dcov[6];
            if (denom2inv != 0) {
                dL_da = denom2inv * (-cc * cc * dcx + 2 * cb * cc * dcy + (denom - ca * cc) * dcz);
                dL_dc = denom2inv * (-ca * ca * dcz + 2 * ca * cb * dcy + (denom - ca * cc) * dcx);
                dL_db = denom2inv * 2 * (cb * cc * dcx - (denom + 2 * cb * cb) * dcy + ca * cb * dcz);
                dcov[0] = (T0[0] * T0[0] * dL_da + T0[0] * T1[0] * dL_db + T1[0] * T1[0] * dL_dc);
                dcov[3] = (T0[1] * T0[1] * dL_da + T0[1] * T1[1] * dL_db + T1[1] * T1[1] * dL_dc);
                dcov[5] = (T0[2] * T0[2] * dL_da + T0[2] * T1[2] * dL_db + T1[2] * T1[2] * dL_dc);
                dcov[1] = 2 * T0[0] * T0[1] * dL_da + (T0[0] * T1[1] + T0[1] * T1[0]) * dL_db + 2 * T1[0] * T1[1] * dL_dc;
                dcov[2] = 2 * T0[0] * T0[2] * dL_da + (T0[0] * T1[2] + T0[2] * T1[0]) * dL_db + 2 * T1[0] * T1[2] * dL_dc;
                dcov[4] = 2 * T0[2] * T0[1] * dL_da + (T0[1] * T1[2] + T0[2] * T1[1]) * dL_db + 2 * T1[1] * T1[2] * dL_dc;
            } else {
#pragma unroll
                for (int k = 0; k < 6; k++) dcov[k] = 0.f;
            }
#pragma unroll
            for (int k = 0; k < 6; k++) o_cov[k] = dcov[k];
            float dT0[3], dT1[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                dT0[k] = 2 * p[k] * dL_da + qv[k] * dL_db;
                dT1[k] = 2 * qv[k] * dL_dc + p[k] * dL_db;
            }
            const float dJ00 = vm[0] * dT0[0] + vm[4] * dT0[1] + vm[8] * dT0[2];
            const float dJ02 = vm[2] * dT0[0] + vm[6] * dT0[1] + vm[10] * dT0[2];
            const float dJ11 = vm[1] * dT1[0] + vm[5] * dT1[1] + vm[9] * dT1[2];
            const float dJ12 = vm[2] * dT1[0] + vm[6] * dT1[1] + vm[10] * dT1[2];
            const float tz = 1.f / tzv, tz2 = tz * tz, tz3 = tz2 * tz;
            const float dtx = x_grad_mul * -h_x * tz2 * dJ02;
            const float dty = y_grad_mul * -h_y * tz2 * dJ12;
            const float dtz = -h_x * tz2 * dJ00 - h_y * tz2 * dJ11 + (2 * h_x * tx) * tz3 * dJ02 + (2 * h_y * ty) * tz3 * dJ12;
            f3 dmean = {vm[0] * dtx + vm[1] * dty + vm[2] * dtz, vm[4] * dtx + vm[5] * dty + vm[6] * dtz,
                        vm[8] * dtx + vm[9] * dty + vm[10] * dtz};
            // ---- preprocessCUDA backward (backward.cu:346-396) ----
            const float hw = xf_row(proj, 3, mx, my, mz);
            const float m_w = 1.0f / (hw + 0.0000001f);
            const float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
            dmean.x += (proj[0] * m_w - proj[3] * mul1) * dmx + (proj[1] * m_w - proj[3] * mul2) * dmy;
            dmean.y += (proj[4] * m_w - proj[7] * mul1) * dmx + (proj[5] * m_w - proj[7] * mul2) * dmy;
            dmean.z += (proj[8] * m_w - proj[11] * mul1) * dmx + (proj[9] * m_w - proj[11] * mul2) * dmy;
            if (a.shs) {
                const float *cp = a.v.campos;
                // sh_dir's own subtractions, so the two share them (with a separate chain this kernel spills)
                const f3 dir_orig = {__fsub_rn(mx, cp[0]), __fsub_rn(my, cp[1]), __fsub_rn(mz, cp[2])};
                add_dnormvdv(dir_orig, ddir, dmean);
                if (a.dsh) {
                    // accumulated dL/dRGB, already masked where the forward clamped the colour
                    const f3 dRGB = {sm[PB_DCOL + tid * 3], sm[PB_DCOL + tid * 3 + 1], sm[PB_DCOL + tid * 3 + 2]};
                    sh_grad_row<MULTI>(a.v.D, M, RAW ? sm + PB_SHDC + tid * 3 : row, RAW ? row : row + 3,
                                       sh_dir(mx, my, mz, cp[0], cp[1], cp[2]), dRGB, MULTI ? a.dsh_scale : 1.0f, oacc);
                }
            }
            o_m3d[0] = dmean.x;
            o_m3d[1] = dmean.y;
            o_m3d[2] = dmean.z;
            // ---- computeCov3D backward (backward.cu:278-341) ----
            if (a.scales) {
                const float r = q.x, x = q.y, y = q.z, z = q.w;
                const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                                       {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                                       {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
                const float s[3] = {a.v.scale_modifier * sc0, a.v.scale_modifier * sc1, a.v.scale_modifier * sc2};
                const float dS[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                                        {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                                        {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
                float dMt[3][3];
#pragma unroll
                for (int c = 0; c < 3; c++)
#pragma unroll
                    for (int w = 0; w < 3; w++)
                        dMt[w][c] = 2.0f * s[w] * R[0][w] * dS[c][0] + 2.0f * s[w] * R[1][w] * dS[c][1] +
                                    2.0f * s[w] * R[2][w] * dS[c][2];
#pragma unroll
                for (int k = 0; k < 3; k++) o_scl[k] = R[0][k] * dMt[k][0] + R[1][k] * dMt[k][1] + R[2][k] * dMt[k][2];
#pragma unroll
                for (int k = 0; k < 3; k++)
#pragma unroll
                    for (int w = 0; w < 3; w++) dMt[k][w] *= s[k];
                float4 dq;
                dq.x = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
                dq.y = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) -
                       4 * x * (dMt[2][2] + dMt[1][1]);
                dq.z = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) -
                       4 * y * (dMt[2][2] + dMt[0][0]);
                dq.w = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) -
                       4 * z * (dMt[1][1] + dMt[0][0]);
                if (RAW) {
                    // chain rule of the activations: exp -> x s;  normalize -> (g - q <q, g>) / |q_raw|
                    o_scl[0] *= sc0;
                    o_scl[1] *= sc1;
                    o_scl[2] *= sc2;
                    const float qd = q.x * dq.x + q.y * dq.y + q.z * dq.z + q.w * dq.w, inv = __fdiv_rn(1.0f, q_len);
                    dq = make_float4((dq.x - q.x * qd) * inv, (dq.y - q.y * qd) * inv, (dq.z - q.z * qd) * inv,
                                     (dq.w - q.w * qd) * inv);
                }
                o_rot[0] = dq.x;
                o_rot[1] = dq.y;
                o_rot[2] = dq.z;
                o_rot[3] = dq.w;
            } else {
                o_scl[0] = o_scl[1] = o_scl[2] = 0.f;
                o_rot[0] = o_rot[1] = o_rot[2] = o_rot[3] = 0.f;
            }
        }
    }
    // ---- write-out: the small arrays leave as 1-D bulk copies (TMA stores issued by one thread) when the
    // block is full and everything is 16-byte aligned, else through coalesced loops
    const bool out_bulk = a.out_bulk_ok && full;
    float *rec_out = a.rec11;
    if (a.stage_tab) rec_out = a.stage_tab[(int)((long long)blockIdx.x * a.nviews / gridDim.x)];
    if (out_bulk) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (out_bulk) {
        if (tid == 0) {
            bulk_s2g(a.dmeans2D + (size_t)base * 3, sm + PB_O_M2D, PB_T * 12);
            bulk_s2g(a.dcov3D + (size_t)base * 6, sm + PB_O_COV, PB_T * 24);
            if (a.rec11) {
                bulk_s2g(rec_out + (size_t)base * 11, sm + PB_O_R11, PB_T * 44);
            } else {
                bulk_s2g(a.dopacity + base, sm + PB_O_OPA, PB_T * 4);
                bulk_s2g(a.dmeans3D + (size_t)base * 3, sm + PB_O_M3D, PB_T * 12);
                bulk_s2g(a.dscales + (size_t)base * 3, sm + PB_O_SCL, PB_T * 12);
                bulk_s2g(a.drots + (size_t)base * 4, sm + PB_O_ROT, PB_T * 16);
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    } else {
        pb_flush(a.dmeans2D + (size_t)base * 3, sm + PB_O_M2D, n * 3);
        pb_flush(a.dcov3D + (size_t)base * 6, sm + PB_O_COV, n * 6);
        if (a.rec11) {
            pb_flush(rec_out + (size_t)base * 11, sm + PB_O_R11, n * 11);
        } else {
            pb_flush(a.dopacity + base, sm + PB_O_OPA, n);
            pb_flush(a.dmeans3D + (size_t)base * 3, sm + PB_O_M3D, n * 3);
            pb_flush(a.dscales + (size_t)base * 3, sm + PB_O_SCL, n * 3);
            pb_flush(a.drots + (size_t)base * 4, sm + PB_O_ROT, n * 4);
        }
    }
    if (RAW && a.dsh && M > 0) {
        // the gradient blocks of a CTA are contiguous in both arrays: two bulk stores (or two plain loops)
        if (out_bulk) {
            if (tid == 0) {
                bulk_s2g(a.dsh + (size_t)base * 3, sm + PB_SHDC, PB_T * 12);
                if (M > 1) bulk_s2g(a.dsh_rest + (size_t)base * row_f, sm + PB_SH, PB_T * (uint32_t)row_f * 4);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        } else {
            pb_flush(a.dsh + (size_t)base * 3, sm + PB_SHDC, n * 3);
            pb_flush(a.dsh_rest + (size_t)base * row_f, sm + PB_SH, n * row_f);
        }
    } else if (a.dsh && M > 0) {
        float *dst = a.dsh + (size_t)base * row_f;
        if (a.shs) {
            if (a.sh_vec)
                sh_rows_walk<PB_T, 4>(n, row_f, a.sh_stride,
                                      [&](int g, int s) { *(float4 *)(dst + g) = *(const float4 *)(s_sh + s); });
            else
                sh_rows_walk<PB_T, 1>(n, row_f, a.sh_stride, [&](int g, int s) { dst[g] = s_sh[s]; });
        } else {
            for (int k = tid; k < n * row_f; k += PB_T) dst[k] = 0.f;
        }
    }
    // the bulk stores read shared memory asynchronously: it must stay valid until they have
    if (out_bulk && tid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

static int set_backward_attributes()
{
    SGR_CUDA(cudaFuncSetAttribute(blend_backward_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)BWD_SMEM_BYTES));
    SGR_CUDA(cudaFuncSetAttribute(blend_backward_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)BWD_SMEM_BYTES));
    SGR_CUDA(cudaFuncSetAttribute(blend_backward_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)BWD_SMEM_BYTES_FEAT));
    SGR_CUDA(cudaFuncSetAttribute(blend_backward_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)BWD_SMEM_BYTES_FEAT));
    SGR_CUDA(cudaFuncSetAttribute(preprocess_backward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  200 * 1024));
    SGR_CUDA(cudaFuncSetAttribute(preprocess_backward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  200 * 1024));
    SGR_CUDA(cudaFuncSetAttribute(preprocess_backward_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  200 * 1024));
    return SGR_OK;
}
static DeviceOnce g_backward_attributes;

static void launch_blend_backward(const ViewConsts &v, int P, const ImageState &img, const BinState &bin,
                                  const GeomState &geom, const float *dL_dout_color, float *gacc, float *dL_dcolors,
                                  const FeatureChannel *feat, cudaStream_t st)
{
    const bool packed = ids_packed(P);
    const auto kernel = feat ? (packed ? &blend_backward_kernel<true, true> : &blend_backward_kernel<false, true>)
                             : (packed ? &blend_backward_kernel<true, false> : &blend_backward_kernel<false, false>);
    kernel<<<v.gx * v.gy, 256, feat ? BWD_SMEM_BYTES_FEAT : BWD_SMEM_BYTES, st>>>(
        img.tile_order, img.tile_start, img.tile_cursor, bin.plist, geom.rec, v.W, v.H, v.gx, v.bg, img.final_T,
        img.n_contrib, dL_dout_color, gacc, dL_dcolors, feat ? feat->values : nullptr, feat ? feat->bg : nullptr,
        feat ? feat->dL_dout : nullptr, feat ? feat->dL_dvalues : nullptr);
}

int launch_backward(const SgrView *view, const SgrGaussians *g, const int32_t *radii, const void *geom_buffer,
                    const void *binning_buffer, const void *image_buffer, int64_t num_rendered,
                    const float *dL_dout_color, float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity,
                    float *dL_dmeans3D, float *dL_dcov3D, float *dL_dsh, float *dL_dscales, float *dL_drotations,
                    void *grad_scratch, cudaStream_t st, const SgrBackwardPlan *plan, const FeatureChannel *feat)
{
    const int P = g->P, W = view->image_width, H = view->image_height;
    Layout geom_l(geom_buffer), img_l(image_buffer), bin_l(binning_buffer), scratch_l(grad_scratch);
    GeomState geom = GeomState::carve(geom_l, P);
    ImageState img = ImageState::carve(img_l, W, H);
    BinState bin = BinState::carve(bin_l, (size_t)num_rendered);
    float *gacc = carve_grad_acc(scratch_l, P);
    const SgrStageHook hook = plan ? plan->hook : nullptr;
    void *hook_ctx = plan ? plan->hook_ctx : nullptr;
    float *rec11 = plan ? plan->reduce_records : nullptr;
    // the peer exchange (SgrPeerPlan); MULTI: the pass sums every rank's SH gradient into dL_dsh, see PreBwdArgs::view_tab
    const SgrPeerPlan *pp = plan ? plan->peer : nullptr;
    const bool multi = pp && pp->peer_view_blocks && dL_dsh && g->shs;
    PeerBackward peer{pp, st, P, dL_dmeans3D, dL_dopacity, dL_dscales, dL_drotations};
    const ViewConsts v = view_consts(view, g->M);
    int rc = once_per_device(g_backward_attributes, set_backward_attributes);
    if (rc) return rc;
    // the blend accumulators: 32 B per Gaussian of scratch + the dL_dcolors output itself
    SGR_CUDA(cudaMemsetAsync(gacc, 0, (size_t)P * 32, st));
    SGR_CUDA(cudaMemsetAsync(dL_dcolors, 0, (size_t)P * 12, st));
    if (feat) SGR_CUDA(cudaMemsetAsync(feat->dL_dvalues, 0, (size_t)P * 4, st));
    if (num_rendered > 0)
        SGR_LAUNCH(K_BLEND_BWD, st, launch_blend_backward(v, P, img, bin, geom, dL_dout_color, gacc, dL_dcolors, feat, st));
    // dL_dcolors is final here (with SH colours: the clamp-masked dL/dRGB, i.e. this view's SH factor)
    if (hook) hook(hook_ctx, SGR_STAGE_BLEND_DONE);
    rc = peer.blend_done(multi);
    if (rc) return rc;
    PreBwdArgs a;
    a.means = g->means3D;
    a.scales = g->scales;
    a.rots = g->rotations;
    a.shs = g->shs;
    a.cov_pre = g->cov3D_precomp;
    a.sh_jac = geom.sh_jac;
    a.v = v;
    a.radii = radii;
    a.gacc = gacc;
    a.dcol = dL_dcolors;
    a.dmeans2D = dL_dmeans2D;
    a.dopacity = dL_dopacity;
    a.dmeans3D = dL_dmeans3D;
    a.dcov3D = dL_dcov3D;
    a.dsh = dL_dsh;
    a.dscales = dL_dscales;
    a.drots = dL_drotations;
    a.rec11 = rec11;
    a.view_tab = multi ? (const float *const *)pp->peer_view_blocks : nullptr;
    a.stage_tab = multi ? (float *const *)pp->peer_record_stages : nullptr;
    a.nviews = multi ? pp->peer_nranks : 1;
    a.my_view = multi ? pp->peer_rank : 0;
    a.campos_off = (size_t)3 * P;
    a.dsh_scale = multi ? pp->peer_dsh_scale : 1.0f;
    const bool raw = g->activations != 0;
    a.rec = geom.rec;
    a.dsh_rest = plan ? plan->dL_dsh_rest : nullptr;
    // (the SH arrays are not read; sh_jac is 256-byte aligned by GeomState::carve)
    a.in_bulk_ok = aligned16(gacc) && aligned16(dL_dcolors) && aligned16(g->means3D) &&
                   (!g->scales || aligned16(g->scales)) && (!g->rotations || aligned16(g->rotations)) &&
                   (!g->cov3D_precomp || aligned16(g->cov3D_precomp));
    a.out_bulk_ok = aligned16(dL_dmeans2D) && aligned16(dL_dcov3D) &&
                    (rec11 ? aligned16(rec11)
                           : (aligned16(dL_dopacity) && aligned16(dL_dmeans3D) && aligned16(dL_dscales) &&
                              aligned16(dL_drotations)));
    if (raw && g->shs && dL_dsh)
        a.out_bulk_ok = a.out_bulk_ok && aligned16(dL_dsh) && (g->M == 1 || aligned16(a.dsh_rest));
    a.sh_stride = 0;
    a.sh_vec = 0;
    if (g->shs && !raw) a.sh_stride = sh_row_stride(g->M, aligned16(dL_dsh), &a.sh_vec);  // rows leave as 16-byte stores
    // the SH block: dL/dsh rows, and before them the Jacobian rows (9 floats per Gaussian, M = 1 has shorter rows)
    int sh_block = raw ? (g->M > 0 ? (g->M - 1) * 3 : 0) : a.sh_stride;
    if (g->shs && sh_block < 9) sh_block = 9;
    a.pf_off = PB_SH + PB_T * sh_block;
    const int pulled = a.view_tab ? (a.nviews - 1 < PB_VB ? a.nviews - 1 : PB_VB) : 0;
    const size_t dyn = (size_t)(a.pf_off + pulled * PB_T * 3) * sizeof(float) + 16;
    // the per-Gaussian pass, in `num_chunks` Gaussian ranges (multiples of the CTA size) so that a caller
    // can start reducing a finished range while the next one is computed
    const int nchunks = backward_chunks(P, plan ? plan->num_chunks : 1);
    const int blocks = (P + PB_T - 1) / PB_T;
    const auto preprocess = raw ? &preprocess_backward_kernel<true>
                                : a.view_tab ? &preprocess_backward_kernel<false, true> : &preprocess_backward_kernel<false>;
    for (int c = 0; c < nchunks; c++) {
        int b0, b1;
        chunk_blocks(blocks, nchunks, c, plan ? plan->chunk_taper : 0, &b0, &b1);
        a.p0 = b0 * PB_T;
        a.p1 = min(P, b1 * PB_T);
        if (b1 > b0) SGR_LAUNCH(K_PRE_BWD, st, preprocess<<<b1 - b0, PB_T, dyn, st>>>(a));
        if (hook) hook(hook_ctx, SGR_STAGE_CHUNK_DONE + c);
        rc = peer.chunk_done(c, a.p0, a.p1);
        if (rc) return rc;
    }
    rc = peer.finish();
    if (rc) return rc;
    SGR_CUDA(cudaGetLastError());
    if (view->debug) SGR_CUDA(cudaStreamSynchronize(st));
    return SGR_OK;
}

}  // namespace sgr
