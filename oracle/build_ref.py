"""Compile the UNMODIFIED reference CUDA rasterizer for sm_90a into oracle/_ref/.

The sources are compiled where they lie under /root/reference (never copied into the repo);
only build products go to oracle/_ref/ (git-ignored, but shipped to the GPU box by gpurun):

    oracle/_ref/diff_gaussian_rasterization/_C.so        <- the 5 reference translation units
    oracle/_ref/diff_gaussian_rasterization/__init__.py  <- installed copy of the reference's
                                                            own Python wrapper (like pip --target)

Flags follow the reference's setup.py (DGR/setup.py:29: no arch flags, no fast-math) plus
`-gencode arch=compute_90a,code=sm_90a` and `-include cstdint` (gcc 13 needs it for
rasterizer_impl.h; no source edit).  This is the parity oracle on the GPU and the
"reference CUDA build on 1xH100" baseline of bench.py --impl reference.
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/gaussian_splatting/submodules/diff-gaussian-rasterization"
OUT = os.path.join(HERE, "_ref", "diff_gaussian_rasterization")


def main() -> int:
    if not os.path.isdir(REF):
        print(f"[build_ref] {REF} not present (GPU box?) - using prebuilt oracle/_ref if any")
        return 0
    so = os.path.join(OUT, "_C.so")
    srcs = [os.path.join(REF, p) for p in (
        "cuda_rasterizer/rasterizer_impl.cu", "cuda_rasterizer/forward.cu",
        "cuda_rasterizer/backward.cu", "rasterize_points.cu", "ext.cpp")]
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(s) for s in srcs):
        print("[build_ref] up to date:", so)
        return 0
    os.makedirs(OUT, exist_ok=True)
    build_dir = os.path.join(HERE, "_ref", "_build")
    os.makedirs(build_dir, exist_ok=True)
    from torch.utils import cpp_extension
    cpp_extension.load(
        name="_C",
        sources=srcs,
        extra_include_paths=[os.path.join(REF, "third_party/glm"), REF],
        extra_cflags=["-O3", "-include", "cstdint"],
        extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a", "-include", "cstdint"],
        build_directory=build_dir,
        with_cuda=True,
        is_python_module=False,
        verbose=True,
    )
    shutil.copyfile(os.path.join(build_dir, "_C.so"), so)
    shutil.copyfile(os.path.join(REF, "diff_gaussian_rasterization", "__init__.py"),
                    os.path.join(OUT, "__init__.py"))
    print("[build_ref] built", so)
    return 0


if __name__ == "__main__":
    sys.exit(main())
