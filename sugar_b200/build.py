"""Build libsugar_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a.

    python sugar_b200/build.py        # or sugar_b200.build.build_library()

The .so is git-ignored; __graft_entry__.build() compiles it (nvcc cross-compiles for sm_90a without a
GPU).  No torch headers are involved: the boundary is plain C (include/sugar_b200.h).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("SGR_LIB_OUT", os.path.join(HERE, "lib", "libsugar_b200.so"))
SOURCES = ["sgr_api.cu", "sgr_forward.cu", "sgr_backward.cu", "sgr_exchange.cu", "sgr_field.cu", "sgr_normal.cu", "sgr_knn.cu", "sgr_scan.cu", "sgr_meshbind.cu",
           "sgr_peer.cu", "sgr_loss.cu", "sgr_meshloss.cu", "sgr_meshlap.cu", "sgr_splatmesh.cu",
           "sgr_texture.cu", "sgr_mcubes.cu", "sgr_decimate.cu", "sgr_densify.cu", "sgr_poisson.cu", "sgr_compose.cu",
           "sgr_postprocess.cu", "sgr_adam.cu", "sgr_image.cu", "sgr_lpips.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--shared",
]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "sugar_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; libsugar_b200.so must be prebuilt (it travels with the repo snapshot)")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "lib", src.replace(".cu", ".o"))
        obj = obj if "SGR_LIB_OUT" not in os.environ else LIB + "." + src.replace(".cu", ".o")
        cmd = [nvcc] + [f for f in NVCC_FLAGS if f != "--shared"] + os.environ.get("SGR_NVCC_EXTRA", "").split() + \
              ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            print(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {src}")
    subprocess.check_call([nvcc, "--shared", "-o", LIB] + objs + ["-Xcompiler", "-fPIC"])
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
