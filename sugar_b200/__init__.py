"""sugar_b200 -- Hopper (sm_90a) rasterizer + density-field hot path for Anttwo/SuGaR.

    sugar_b200.diff_gaussian_rasterization   drop-in for the reference's rasterizer module
    sugar_b200.field                         fused SuGaR density / SDF field (get_field_values)
    sugar_b200.parallel                      view-sharded multi-GPU step (NCCL all-reduce of grads)
    sugar_b200.scenes                        seeded synthetic clouds / cameras for tests and bench

Importing this package loads libsugar_b200.so and fails loudly when it is missing: there is no
CPU or PyTorch fallback.
"""
import sys

from . import _lib  # noqa: F401  (raises if the CUDA library is absent)

__all__ = ["install"]


def install() -> None:
    """Make `import diff_gaussian_rasterization` resolve to the sugar_b200 implementation."""
    from . import diff_gaussian_rasterization as dgr
    sys.modules["diff_gaussian_rasterization"] = dgr
