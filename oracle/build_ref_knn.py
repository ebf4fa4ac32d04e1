"""Compile the UNMODIFIED reference simple-knn (distCUDA2) for sm_90a into oracle/_ref/simple_knn/.

The companion of build_ref.py: the sources are compiled where they lie under /root/reference (never copied into the
repo); only build products go to oracle/_ref/ (git-ignored, but shipped to the GPU box with the tree):

    oracle/_ref/simple_knn/simple_knn_C.so   <- spatial.cu, simple_knn.cu, ext.cpp

The extension is named `simple_knn_C`, not the reference's `simple_knn._C`, so that it can never be mistaken for an
installed simple-knn nor collide with the rasterizer's `_C` in torch's extension registry.  Import it with
oracle/_ref/simple_knn on sys.path, after torch: `import simple_knn_C; simple_knn_C.distCUDA2(points)`.

Flags follow the reference's setup.py (no arch flags, no fast-math) plus `-gencode arch=compute_90a,code=sm_90a` and
`-include cfloat` (simple_knn.cu uses FLT_MAX without including it; current toolchains no longer pull it in; no
source edit).
This is the golden source of tests/golden/make_refbuild_distcuda2_golden.py and the baseline of
scripts/bench_pretrain.py.
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/gaussian_splatting/submodules/simple-knn"
OUT = os.path.join(HERE, "_ref", "simple_knn")
NAME = "simple_knn_C"


def main() -> int:
    if not os.path.isdir(REF):
        print(f"[build_ref_knn] {REF} not present (GPU box?) - using prebuilt oracle/_ref if any")
        return 0
    so = os.path.join(OUT, NAME + ".so")
    srcs = [os.path.join(REF, p) for p in ("spatial.cu", "simple_knn.cu", "ext.cpp")]
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(s) for s in srcs):
        print("[build_ref_knn] up to date:", so)
        return 0
    os.makedirs(OUT, exist_ok=True)
    build_dir = os.path.join(HERE, "_ref", "_build_simple_knn")
    os.makedirs(build_dir, exist_ok=True)
    from torch.utils import cpp_extension
    cpp_extension.load(
        name=NAME,
        sources=srcs,
        extra_include_paths=[REF],
        extra_cflags=["-O3"],
        extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a", "-include", "cfloat"],
        build_directory=build_dir,
        with_cuda=True,
        is_python_module=False,
        verbose=True,
    )
    shutil.copyfile(os.path.join(build_dir, NAME + ".so"), so)
    print("[build_ref_knn] built", so)
    return 0


if __name__ == "__main__":
    sys.exit(main())
