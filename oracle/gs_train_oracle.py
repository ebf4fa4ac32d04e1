"""The vanilla 3DGS trainer's per-iteration decisions (gaussian_splatting/train.py:51-128) restated as the loop
writes them, with OptimizationParams' defaults (arguments/__init__.py:73-89).  train.gs_phase must agree with it."""


class _Gaussians:
    def __init__(self, max_sh_degree):
        self.active_sh_degree, self.max_sh_degree = 0, max_sh_degree

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1


def decisions(iterations=30_000, max_sh_degree=3, sh_every=1000, densify_from_iter=500, densify_until_iter=15_000,
              densification_interval=100, opacity_reset_interval=3000, white_background=False):
    """-> {iteration: dict} for iterations 1..`iterations`, each with the keys train.gs_phase uses: "sh_degree", and
    "stats", "densify" (with "size_threshold"), "reset_opacity", "step" when they happen.  `sh_every` is the
    reference's literal 1000, a parameter here so that scaled-down schedules can be checked too."""
    gaussians = _Gaussians(max_sh_degree)
    out = {}
    for iteration in range(1, iterations + 1):
        ev = {}
        if iteration % sh_every == 0:
            gaussians.oneupSHdegree()
        ev["sh_degree"] = gaussians.active_sh_degree
        if iteration < densify_until_iter:
            ev["stats"] = True
            if iteration > densify_from_iter and iteration % densification_interval == 0:
                ev["densify"] = True
                ev["size_threshold"] = 20 if iteration > opacity_reset_interval else None
            if iteration % opacity_reset_interval == 0 or (white_background and iteration == densify_from_iter):
                ev["reset_opacity"] = True
        if iteration < iterations:
            ev["step"] = True
        out[iteration] = ev
    return out
