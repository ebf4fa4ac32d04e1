"""Edited and composited renders of refined models: SuGaRCompositor (sugar_scene/sugar_compositor.py:29-244) with the
editable bound model (sugar_model.py:562-667) behind it.

After refinement a user deforms the bound mesh (poses it, animates it) and places several models in one scene.  A
`Composition` holds the parts once; each `render` call is one frame:

    comp = Composition([dict(verts=ref_verts, faces=faces, bary=bary, scales_raw=_scales, complex_raw=_quaternions,
                             thickness=surface_mesh_thickness, densities=all_densities, sh=sh_coordinates),
                        dict(points=..., scaling=..., quaternions=..., opacities=..., sh=..., idx=rows_to_render)])
    image = comp.render(c2w, fov_x, fov_y, H, W, verts=[posed_verts, None], sh_rotations=[None, R])   # [H, W, 3]

A bound part's Gaussians are rebuilt every frame by one `sgr_meshbind_edited_forward` launch from the frame's vertices,
written straight into the composite buffers (at the part's offset, or through an `out_rows` map when `idx` selects rows).
Everything else -- opacities, SH, plain parts' geometry -- is gathered once at construction.  A frame is one rasterizer
call; with an `sh_rotations` entry, colours come from one `sgr_sh_colors_rotated` launch over the composite (identity for
parts without a rotation) instead of the rasterizer's in-kernel SH.  Forward only: frames run under no_grad and make no
host synchronisation when c2w and the rotations are host tensors or arrays.

Deliberate differences from the reference compositor: positions come from the parts (the reference takes one
`positions` tensor from the caller), and an sh_rotation applies to the rows actually rendered (the reference forms the
rotated directions from `positions` before selecting idx_to_render).  Not built: compute_covariance_in_rasterizer=False,
use_same_scale_in_all_directions, gradients.
"""
import math

import torch

from . import meshbind
from ._lib import check, lib, require_cuda, stream, tensor
from .diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
from .render import camera_matrices

_BOUND = ("verts", "faces", "bary", "scales_raw", "complex_raw", "thickness", "densities", "sh")
_PLAIN = ("points", "scaling", "quaternions", "opacities", "sh")


def _no_grad_input(name, t):
    if torch.is_grad_enabled() and t.requires_grad:
        raise ValueError(f"{name} requires grad: a composition is forward only")


def _rows(part, name, P, dev):
    """The part's rows to render, checked on the host: int64 [N] in [0, P), no repeats (each Gaussian has one row)."""
    idx = part.get("idx")
    if idx is None:
        return None
    idx = tensor(idx, f"{name}.idx", torch.int64, ("N",), dev)
    if idx.numel():
        lo, hi, uniq = int(idx.min()), int(idx.max()), int(torch.unique(idx).numel())
        if lo < 0 or hi >= P:
            raise ValueError(f"{name}.idx holds rows outside [0, {P})")
        if uniq != idx.numel():
            raise ValueError(f"{name}.idx repeats a row")
    return idx


def _pinned_to(t, dev):
    """A host tensor to `dev` without a host synchronisation: staged through pinned memory, copied asynchronously."""
    return t.contiguous().pin_memory().to(dev, non_blocking=True)


def sh_colors_rotated(points, sh, campos, group_start, group_rot, sh_degree):
    """Colours [P,3] of SH rows `sh` [P,M,3] at `points` [P,3] seen from `campos` [3] with the view direction turned by
    the row's group rotation: clamp_min(eval_sh(normalize(p - campos) @ R_g) + 0.5, 0), the compositor's sh_rotations
    colour in the rasterizer's own SH basis.  group_start int64 [G+1] (0 .. P), group_rot float32 [G,3,3] or [G,9].
    All CUDA tensors on one device."""
    points = tensor(points, "points", torch.float32, ("P", 3))
    dev, P = points.device, points.shape[0]
    sh = tensor(sh, "sh", torch.float32, (P, "M", 3), dev)
    campos = tensor(campos.reshape(-1), "campos", torch.float32, (3,), dev, "points")
    group_start = tensor(group_start, "group_start", torch.int64, ("G+1",), dev, "points")
    G = group_start.shape[0] - 1
    group_rot = tensor(group_rot.reshape(-1, 9), "group_rot", torch.float32, (G, 9), dev, "points")
    if not 0 <= sh_degree <= 3 or sh.shape[1] < (sh_degree + 1) ** 2:
        raise ValueError(f"SH degree {sh_degree} needs (degree + 1)^2 <= M = {sh.shape[1]} coefficients, degree <= 3")
    require_cuda("compose", points)
    colors = torch.empty((P, 3), device=dev)
    _colors_launch(P, sh.shape[1], sh_degree, points, sh, campos, G, group_start, group_rot, colors)
    return colors


def _colors_launch(P, M, deg, points, sh, campos, G, group_start, group_rot, colors):
    with torch.cuda.device(points.device):
        check(lib.sgr_sh_colors_rotated(P, M, deg, points.data_ptr(), sh.data_ptr(), campos.data_ptr(), G,
                                        group_start.data_ptr(), group_rot.data_ptr(), colors.data_ptr(),
                                        stream(points.device)))


class Composition:
    """Several refined models rendered together, each bound model at its own (edited) vertices.  `parts` is a list of
    dicts: a bound refined model (keys verts = the reference vertices it was made editable at, faces, bary, scales_raw,
    complex_raw, thickness, densities [P,1] (raw: rendered as sigmoid), sh [P,M,3]) or a plain, activated Gaussian set
    (points, scaling, quaternions, opacities [P,1], sh [P,M,3]).  Either may carry idx (int64 rows to render, in that
    order).  Construction checks every part (ValueError) and gathers the static rows into the composite buffers."""

    def __init__(self, parts):
        parts = list(parts)
        if not parts:
            raise ValueError("a composition needs at least one part")
        dev, M, self._bound, static, sizes = None, None, [], [], []
        for i, part in enumerate(parts):
            name = f"parts[{i}]"
            bound = "faces" in part
            missing = [k for k in (_BOUND if bound else _PLAIN) if k not in part]
            if missing:
                raise ValueError(f"{name} lacks {missing}")
            if bound:
                a = meshbind.edited_args(part["verts"], part["verts"], part["faces"], part["bary"], part["scales_raw"],
                                         part["complex_raw"], part["thickness"])
                if dev is not None and a.verts.device != dev:
                    raise ValueError(f"{name}.verts on {a.verts.device}, parts[0] on {dev}")
                dev, P = a.verts.device, a.P
                dens = tensor(part["densities"], f"{name}.densities", torch.float32, (P, 1), dev, "parts[0]")
                _no_grad_input(f"{name}.densities", dens)
                cols = dict(opacities=torch.sigmoid(dens))
            else:
                pts = tensor(part["points"], f"{name}.points", torch.float32, ("P", 3), dev, "parts[0]")
                dev, P = pts.device, pts.shape[0]
                cols = dict(points=pts)
                for k, w in (("scaling", 3), ("quaternions", 4), ("opacities", 1)):
                    cols[k] = tensor(part[k], f"{name}.{k}", torch.float32, (P, w), dev, "parts[0]")
                for k, t in cols.items():
                    _no_grad_input(f"{name}.{k}", t)
            sh = tensor(part["sh"], f"{name}.sh", torch.float32, (P, "M", 3), dev, "parts[0]")
            _no_grad_input(f"{name}.sh", sh)
            if M is not None and sh.shape[1] != M:
                raise ValueError(f"{name}.sh has {sh.shape[1]} SH coefficients, parts[0].sh {M}")
            M = sh.shape[1]
            cols["sh"] = sh
            idx = _rows(part, name, P, dev)
            sizes.append(P if idx is None else idx.numel())
            static.append((cols, idx))
            if bound:
                self._bound.append((i, a, idx))
        require_cuda("compose", *(t for cols, _ in static for t in cols.values()))
        self.device, self.M, self.num_parts = dev, M, len(parts)
        self.starts = [0]
        for n in sizes:
            self.starts.append(self.starts[-1] + n)
        N = self.starts[-1]
        with torch.cuda.device(dev), torch.no_grad():
            self.points = torch.empty((N, 3), device=dev)
            self.scaling = torch.empty((N, 3), device=dev)
            self.quaternions = torch.empty((N, 4), device=dev)
            self.opacities = torch.empty((N, 1), device=dev)
            self.sh = torch.empty((N, M, 3), device=dev)
            self.colors = torch.empty((N, 3), device=dev)
            self.means2D = torch.zeros((N, 3), device=dev)
            self.group_start = torch.tensor(self.starts, dtype=torch.int64).to(dev)
            for (cols, idx), s0, s1 in zip(static, self.starts[:-1], self.starts[1:]):
                for k, t in cols.items():
                    getattr(self, k)[s0:s1] = t if idx is None else t[idx]
            # a bound part with idx writes through out_rows: out_rows[g] = its composite row, -1 when not rendered
            self._out_rows = {}
            for i, a, idx in self._bound:
                if idx is not None:
                    rows = torch.full((a.P,), -1, dtype=torch.int64, device=dev)
                    rows[idx] = torch.arange(self.starts[i], self.starts[i + 1], dtype=torch.int64, device=dev)
                    self._out_rows[i] = rows

    def _frame_args(self, verts):
        """Checked launch arguments of every bound part for this frame's vertices."""
        if verts is not None and len(verts) != self.num_parts:
            raise ValueError(f"verts must hold one entry per part ({self.num_parts}), got {len(verts)}")
        bound = {i for i, _, _ in self._bound}
        for i in range(self.num_parts):
            if verts is not None and verts[i] is not None and i not in bound:
                raise ValueError(f"verts[{i}] given for a part that is not mesh-bound")
        out = []
        for i, a, _ in self._bound:
            v = a.reference_verts if verts is None or verts[i] is None else verts[i]
            out.append((i, meshbind.edited_args(v, a.reference_verts, a.faces, a.bary, a.scales_raw, a.complex_raw,
                                                a.thickness)))
        return out

    def _rotations(self, sh_rotations):
        if sh_rotations is None:
            return None
        if len(sh_rotations) != self.num_parts:
            raise ValueError(f"sh_rotations must hold one entry per part ({self.num_parts}), got {len(sh_rotations)}")
        if all(R is None for R in sh_rotations):
            return None
        rots = []
        for i, R in enumerate(sh_rotations):
            if R is None:
                rots.append(torch.eye(3, device=self.device))
                continue
            R = torch.as_tensor(R, dtype=torch.float32)
            if R.shape != (3, 3):
                raise ValueError(f"sh_rotations[{i}] must be [3, 3], got {tuple(R.shape)}")
            _no_grad_input(f"sh_rotations[{i}]", R)
            rots.append(R.to(self.device) if R.is_cuda else _pinned_to(R, self.device))
        return rots

    def render(self, c2w, fov_x, fov_y, image_height, image_width, verts=None, sh_rotations=None, bg_color=None,
               sh_deg=3, principal_point=(0.0, 0.0)):
        """One frame -> image [H, W, 3].  c2w: [3,4] or [4,4] camera-to-world as render.camera_matrices takes it (a CUDA
        c2w is read back to the host, one synchronisation).  verts[i]: part i's vertices this frame (None: its
        reference vertices).  sh_rotations[i]: [3,3] turning part i's view direction (d @ R) for its SH colour, or
        None."""
        frame = self._frame_args(verts)
        if not 0 <= sh_deg <= 3 or self.M < (sh_deg + 1) ** 2:
            raise ValueError(f"SH degree {sh_deg} needs (degree + 1)^2 <= M = {self.M} coefficients, degree <= 3")
        rots = self._rotations(sh_rotations)
        dev = self.device
        with torch.no_grad(), torch.cuda.device(dev):
            for i, a in frame:
                rows = self._out_rows.get(i)
                if rows is None:
                    s0, s1 = self.starts[i], self.starts[i + 1]
                    meshbind.edited_launch(a, self.points[s0:s1], self.scaling[s0:s1], self.quaternions[s0:s1])
                else:
                    meshbind.edited_launch(a, self.points, self.scaling, self.quaternions, rows)
            c2w = torch.as_tensor(c2w, dtype=torch.float32).cpu()
            world_view, full_proj, campos = (_pinned_to(t, dev) for t in
                                             camera_matrices(c2w, fov_x, fov_y, principal_point=principal_point))
            bg = torch.zeros(3, device=dev) if bg_color is None else torch.as_tensor(bg_color, dtype=torch.float32)
            bg = bg if bg.is_cuda else _pinned_to(bg, dev)
            if rots is None:
                kw = dict(shs=self.sh)
            else:
                _colors_launch(self.points.shape[0], self.M, sh_deg, self.points, self.sh, campos, self.num_parts,
                               self.group_start, torch.stack(rots), self.colors)
                kw = dict(colors_precomp=self.colors)
            settings = GaussianRasterizationSettings(
                image_height=int(image_height), image_width=int(image_width), tanfovx=math.tan(fov_x * 0.5),
                tanfovy=math.tan(fov_y * 0.5), bg=bg, scale_modifier=1., viewmatrix=world_view, projmatrix=full_proj,
                sh_degree=sh_deg, campos=campos, prefiltered=False, debug=False)
            image, _ = GaussianRasterizer(settings)(means3D=self.points, means2D=self.means2D, opacities=self.opacities,
                                                    scales=self.scaling, rotations=self.quaternions, **kw)
        return image.permute(1, 2, 0)
