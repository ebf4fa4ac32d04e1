"""Golden results of the UNMODIFIED reference simple-knn build (oracle/_ref/simple_knn, oracle/build_ref_knn.py) for
tests/test_gpu_pretrain.py:

    python tests/golden/make_refbuild_distcuda2_golden.py [OUT_DIR]      (needs a GPU and the reference build)

writes OUT_DIR (default tests/golden)/refbuild_distcuda2_<cloud>.npz with `dist` = distCUDA2(points) (float32 [P]) for
each cloud of tests/pretrain_cases.py, whose points the tests rebuild from the same seeds.  Each cloud is run twice and
the two results must be identical (the reference has no atomics on this path).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref", "simple_knn"))
import pretrain_cases  # noqa: E402
import simple_knn_C  # noqa: E402


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    for name, pts in pretrain_cases.clouds().items():
        p = pts.cuda()
        a = simple_knn_C.distCUDA2(p).cpu().numpy()
        b = simple_knn_C.distCUDA2(p).cpu().numpy()
        assert a.dtype == np.float32 and a.shape == (pts.shape[0],) and np.array_equal(a.view(np.int32),
                                                                                       b.view(np.int32)), name
        np.savez_compressed(os.path.join(out_dir, f"refbuild_distcuda2_{name}.npz"), dist=a)
        print(name, pts.shape[0], a[:3])


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
