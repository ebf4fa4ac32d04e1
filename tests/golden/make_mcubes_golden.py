"""Golden vectors for the marching-cubes extraction from the reference's OWN code.

Runs in the build container (needs /root/reference):  python tests/golden/make_mcubes_golden.py
The marching-cubes branch of sugar_extractors/coarse_mesh.py needs a trained model, pytorch3d, PyMCubes and open3d.
This script reads exactly coarse_mesh.py:635-664 (foreground) and :675-707 (background) from /root/reference at run
time, dedents the lines and executes them unchanged with these stand-ins:
  * `resolution` injected small (32 and 28) and `surface_levels` = [0.3] (train.py's default);
  * `sugar`: SuGaR.compute_density and SuGaR.get_gaussians_closest_to_samples called unbound, with pytorch3d's
    knn_points restated as an exact cdist + topk, and a fixed get_cameras_spatial_extent;
  * `mcubes`: records the volume it is given and returns oracle/mcubes_oracle.py's marching cubes.
Only the resulting numbers are stored.
Outputs: tests/golden/mcubes_<case>.npz
"""
import os
import sys
import textwrap
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import mcubes_oracle as mo  # noqa: E402
from make_field_golden import import_reference_sugar  # noqa: E402

SRC = "/root/reference/sugar_extractors/coarse_mesh.py"
BLOCKS = ((635, 664), (675, 707))
LEVEL = 0.3


def make_cloud(kind, seed):
    """A shell of Gaussians inside the foreground box; "floaters" adds a few points beyond mean +- 4 sigma and
    Gaussians beyond the foreground box (they give the background grid a surface)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "shell":
        P = 700
        d = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
        pts = 0.55 * d + 0.02 * torch.randn(P, 3, generator=g)
    else:
        P = 900
        pts = 0.25 * torch.randn(P, 3, generator=g)
        pts[:12] = torch.tensor([2.6, -2.2, 1.9]) * (1 + 0.2 * torch.rand(12, 3, generator=g))   # floaters
        pts[12:112] = torch.tensor([1.8, 0.4, -0.3]) + 0.15 * torch.randn(100, 3, generator=g)  # beyond the fg box
    scaling = torch.exp(torch.randn(P, 3, generator=g) * 0.3 + np.log(0.07))
    quats = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    strengths = torch.sigmoid(torch.randn(P, 1, generator=g) + 1.5)
    sh_dc = 0.8 * torch.randn(P, 1, 3, generator=g)
    return pts.float(), scaling.float(), quats.float(), strengths.float(), sh_dc.float()


def knn_cdist(x, y, K):
    d = torch.cdist(x[0].double(), y[0].double(), compute_mode="donot_use_mm_for_euclid_dist")
    return SimpleNamespace(idx=torch.topk(d, K, dim=-1, largest=False, sorted=True).indices[None])


CASES = {"shell_r32": dict(kind="shell", seed=21, R=32, extent=1.0),
         "floaters_r28": dict(kind="floaters", seed=22, R=28, extent=0.9)}


def main():
    sm = import_reference_sugar()
    SuGaR = sm.SuGaR
    sm.knn_points = knn_cdist
    from sugar_utils.spherical_harmonics import SH2RGB
    lines = open(SRC).read().splitlines()
    codes = [compile(textwrap.dedent("\n".join(lines[a - 1:b])), f"coarse_mesh.py:{a}-{b}", "exec") for a, b in BLOCKS]
    for name, cfg in CASES.items():
        pts, scaling, quats, strengths, sh_dc = make_cloud(cfg["kind"], cfg["seed"])

        class Fake:
            device = "cpu"
            points = pts
            _sh_coordinates_dc = sh_dc
            knn_to_track = 16

            def __init__(self):
                self.scaling, self.quaternions, self.strengths = scaling, quats, strengths

            def get_covariance(self, **kw):
                return SuGaR.get_covariance(self, **kw)

            def get_gaussians_closest_to_samples(self, x, n_closest_gaussian=None):
                return SuGaR.get_gaussians_closest_to_samples(self, x, n_closest_gaussian)

            def compute_density(self, x, **kw):
                return SuGaR.compute_density(self, x, **kw)

            def get_cameras_spatial_extent(self):
                return cfg["extent"]

        volumes = []

        class MC:
            @staticmethod
            def marching_cubes(vol, level):
                volumes.append(np.array(vol, copy=True))
                return mo.marching_cubes(vol, level)

        ns = dict(torch=torch, sugar=Fake(), resolution=cfg["R"], surface_levels=[LEVEL], mcubes=MC, SH2RGB=SH2RGB,
                  CONSOLE=SimpleNamespace(print=lambda *a, **k: None), print=lambda *a, **k: None)
        for code in codes:
            exec(code, ns)
        out = dict(points=pts.numpy(), scaling=scaling.numpy(), quaternions=quats.numpy(),
                   strengths=strengths.numpy(), sh_dc=sh_dc.numpy(), extent=np.float64(cfg["extent"]),
                   resolution=np.int64(cfg["R"]), level=np.float64(LEVEL),
                   fg_volume=volumes[0], bg_volume=volumes[1],
                   fg_verts=ns["verts"].numpy(), fg_faces=ns["faces"].numpy().reshape(-1, 3),
                   fg_colors=ns["verts_colors"].numpy(),
                   bg_verts=ns["bg_verts"].numpy(), bg_faces=ns["bg_faces"].numpy().reshape(-1, 3),
                   bg_colors=ns["bg_verts_colors"].numpy())
        print(name, {k: v.shape for k, v in out.items() if hasattr(v, "shape")})
        np.savez_compressed(os.path.join(HERE, f"mcubes_{name}.npz"), **out)


if __name__ == "__main__":
    main()
