// sgr_adam.cu -- one Adam step over every parameter group in one launch (sugar_b200/optim.py, the optimizer of
// SuGaR's trainers: sugar_scene/sugar_optimizer.py, torch.optim.Adam(groups, lr=0.0, eps=1e-15) in torch's default
// foreach form).
//
// adam_step_kernel  one launch over every segment (one segment per parameter tensor), found per CTA from a
//                   first_block[] prefix in a table passed by value, as densify_emit_kernel finds its column.  Each
//                   element is read and written once: param, exp_avg and exp_avg_sq read and written, grad read
//                   (28 B per element).  float4 accesses when the segment's four pointers are 16-byte aligned,
//                   scalar otherwise (a view at any float offset is legal).  No atomics, no shared memory.
//
// The arithmetic is torch's foreach sequence (torch/optim/adam.py, _multi_tensor_adam, the non-capturable branch),
// each op rounded to float32 on its own and in its order, so that a step is bit-identical to torch.optim.Adam's:
//     m = lerp(m, g, 1 - beta1)          _foreach_lerp_     ATen's lerp: m + w (g - m) for |w| < 0.5, else
//                                                            g - (g - m)(1 - w); the product and sum are one fma
//     v = v * beta2                      _foreach_mul_
//     v = v + (1 - beta2) * (g * g)      _foreach_addcmul_  g * g rounded, then one fma
//     d = sqrt(v)                        _foreach_sqrt
//     d = d / bias_correction2_sqrt      _foreach_div_      a true division (not a reciprocal product)
//     d = d + eps                        _foreach_add_
//     p = p + step_size * (m / d)        _foreach_addcdiv_  m / d rounded, then one fma
// torch's foreach kernels are compiled with nvcc's default contraction, which makes each of the three "x + s * y"
// forms one fma; here they are explicit fmaf, and every other op is an _rn intrinsic, which the compiler never
// contracts, so the result does not depend on this file's flags (tests/test_gpu_optim.py holds it to torch's bits
// for both lerp branches).  The host
// computes the scalars from the step count in float64 and rounds them to float32, as the foreach kernels receive
// them (sugar_b200/optim.py).
#include "sgr_internal.cuh"

namespace sgr {

constexpr int ADAM_THREADS = 256;
constexpr int ADAM_PER_THREAD = 4;                              // one float4, or four scalars
constexpr int ADAM_PER_BLOCK = ADAM_THREADS * ADAM_PER_THREAD;   // elements per CTA

struct AdamTable {
    SgrAdamSegment seg[SGR_ADAM_MAX_SEGMENTS];
    unsigned first_block[SGR_ADAM_MAX_SEGMENTS + 1];   // block prefix over the segments
    int vec[SGR_ADAM_MAX_SEGMENTS];                      // all four pointers 16-byte aligned
    int n;
};

struct AdamScalars {
    float w, omw, beta2, omb2, bc2, eps, step;
    bool small;
};

__device__ __forceinline__ void adam_element(const AdamScalars &s, float &p, float g, float &m, float &v)
{
    // at::lerp (ATen/native/Lerp.h): the weight-small branch contracts self + w * (end - self)
    const float d = __fsub_rn(g, m);
    m = s.small ? fmaf(s.w, d, m) : fmaf(-d, s.omw, g);
    v = fmaf(s.omb2, __fmul_rn(g, g), __fmul_rn(v, s.beta2));
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), s.bc2), s.eps);
    p = fmaf(s.step, __fdiv_rn(m, den), p);
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_step_kernel(AdamTable tab)
{
    int c = 0;
    while (c + 1 < tab.n && blockIdx.x >= tab.first_block[c + 1]) c++;
    const SgrAdamSegment seg = tab.seg[c];
    const unsigned n = (unsigned)seg.n;
    AdamScalars s;
    s.w = seg.one_minus_beta1;
    s.small = fabsf(s.w) < 0.5f;
    s.omw = __fsub_rn(1.0f, s.w);
    s.beta2 = seg.beta2;
    s.omb2 = seg.one_minus_beta2;
    s.bc2 = seg.bias_correction2_sqrt;
    s.eps = seg.eps;
    s.step = seg.step_size;
    const unsigned base = (blockIdx.x - tab.first_block[c]) * ADAM_PER_BLOCK;
    float *__restrict__ P = seg.param;
    const float *__restrict__ G = seg.grad;
    float *__restrict__ M = seg.exp_avg;
    float *__restrict__ V = seg.exp_avg_sq;
    if (tab.vec[c]) {
        const unsigned e = base + ADAM_PER_THREAD * threadIdx.x;
        if (e + ADAM_PER_THREAD <= n) {
            float4 p = *reinterpret_cast<const float4 *>(P + e), m = *reinterpret_cast<const float4 *>(M + e),
                   v = *reinterpret_cast<const float4 *>(V + e);
            const float4 g = *reinterpret_cast<const float4 *>(G + e);
            adam_element(s, p.x, g.x, m.x, v.x);
            adam_element(s, p.y, g.y, m.y, v.y);
            adam_element(s, p.z, g.z, m.z, v.z);
            adam_element(s, p.w, g.w, m.w, v.w);
            *reinterpret_cast<float4 *>(P + e) = p;
            *reinterpret_cast<float4 *>(M + e) = m;
            *reinterpret_cast<float4 *>(V + e) = v;
        } else {
            for (unsigned k = e; k < n && k < e + ADAM_PER_THREAD; k++) {   // the segment's last < 4 elements
                float p = P[k], m = M[k], v = V[k];
                adam_element(s, p, G[k], m, v);
                P[k] = p, M[k] = m, V[k] = v;
            }
        }
        return;
    }
#pragma unroll
    for (int u = 0; u < ADAM_PER_THREAD; u++) {
        const unsigned k = base + u * ADAM_THREADS + threadIdx.x;
        if (k < n) {
            float p = P[k], m = M[k], v = V[k];
            adam_element(s, p, G[k], m, v);
            P[k] = p, M[k] = m, V[k] = v;
        }
    }
}

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_adam_step(int32_t n_segs, const SgrAdamSegment *segs, void *stream)
{
    if (n_segs < 0 || n_segs > SGR_ADAM_MAX_SEGMENTS || (n_segs > 0 && !segs)) {
        set_error("sgr_adam_step: n_segs=%d (0..%d, segs on the host)", n_segs, SGR_ADAM_MAX_SEGMENTS);
        return SGR_EINVAL;
    }
    AdamTable tab;
    tab.n = n_segs;
    tab.first_block[0] = 0;
    long long blocks = 0;
    for (int c = 0; c < n_segs; c++) {
        const SgrAdamSegment &k = segs[c];
        if (k.n < 0 || k.n > INT32_MAX) {
            set_error("sgr_adam_step: segment %d: n=%lld (0 <= n <= 2^31 - 1)", c, (long long)k.n);
            return SGR_EINVAL;
        }
        if (k.n > 0 && (!k.param || !k.grad || !k.exp_avg || !k.exp_avg_sq)) {
            set_error("sgr_adam_step: segment %d: null pointer", c);
            return SGR_EINVAL;
        }
        tab.seg[c] = k;
        tab.vec[c] = (((size_t)k.param | (size_t)k.grad | (size_t)k.exp_avg | (size_t)k.exp_avg_sq) & 15) == 0;
        blocks += (k.n + ADAM_PER_BLOCK - 1) / ADAM_PER_BLOCK;
        tab.first_block[c + 1] = (unsigned)blocks;
    }
    if (blocks == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st, adam_step_kernel<<<(unsigned)blocks, ADAM_THREADS, 0, st>>>(tab));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
