// sgr_postprocess.cu -- border-face erosion of the refined mesh (postprocess_mesh, sugar_b200/postprocess.py).
//
// The reference (sugar_extractors/refined_mesh.py:140-147) peels the mesh's open borders round by round: a live face
// stays when each of its three edges occurs at least twice among the live faces' (face, edge) entries, found there
// with a K = 2 nearest-neighbour search over the edges' vertex ids.  Here the entries are grouped once into runs of
// equal edges (the caller sorts them, sugar_b200/postprocess.py), and each round is one launch with one thread per
// face that reads the mask of round t and writes that of round t + 1.  A thread walks each of its runs until it has
// seen two live entries, so a run of any length (a non-manifold fan) is handled; a face's own two entries on one
// edge (a repeated vertex id) count as two, as in the reference.  No atomics: the result is deterministic.
#include "sgr_internal.cuh"

namespace sgr {

__global__ void __launch_bounds__(256) border_peel_kernel(int F, const int32_t *__restrict__ entry_run,
                                                          const int32_t *__restrict__ run_ptr,
                                                          const int32_t *__restrict__ run_faces,
                                                          const uint8_t *__restrict__ live,
                                                          uint8_t *__restrict__ next)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    bool keep = live[f] != 0;
#pragma unroll
    for (int m = 0; m < 3 && keep; m++) {
        const int r = entry_run[3 * (size_t)f + m];
        const int end = run_ptr[r + 1];
        int seen = 0;
        for (int j = run_ptr[r]; j < end && seen < 2; j++) seen += live[run_faces[j]] != 0;
        keep = seen >= 2;
    }
    next[f] = keep;
}

}  // namespace sgr

using namespace sgr;

extern "C" int sgr_border_peel(int32_t F, int32_t iterations, const int32_t *entry_run, const int32_t *run_ptr,
                               const int32_t *run_faces, uint8_t *mask, uint8_t *mask_tmp, void *stream)
{
    if (F < 0 || F > INT32_MAX / 3 || iterations < 0 ||
        (F > 0 && iterations > 0 && (!entry_run || !run_ptr || !run_faces || !mask || !mask_tmp || mask == mask_tmp))) {
        set_error("bad arguments to sgr_border_peel: need 0 <= F <= (2^31 - 1) / 3, iterations >= 0, non-null "
                  "tables and two distinct masks (F = %d, iterations = %d)", F, iterations);
        return SGR_EINVAL;
    }
    if (F == 0 || iterations == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    uint8_t *buf[2] = {mask, mask_tmp};
    for (int t = 0; t < iterations; t++) {
        SGR_LAUNCH(K_MISC, st,
                   border_peel_kernel<<<(F + 255) / 256, 256, 0, st>>>(F, entry_run, run_ptr, run_faces, buf[t & 1],
                                                                       buf[(t + 1) & 1]));
        SGR_CUDA(cudaGetLastError());
    }
    if (iterations & 1) SGR_CUDA(cudaMemcpyAsync(mask, mask_tmp, (size_t)F, cudaMemcpyDeviceToDevice, st));
    return SGR_OK;
}
