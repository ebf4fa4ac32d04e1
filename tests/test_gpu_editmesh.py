"""The editable bound model and the compositor on the GPU (sugar_b200/meshbind.py bind_to_edited_mesh,
sugar_b200/compose.py, csrc/sgr_meshbind.cu, csrc/sgr_compose.cu): against goldens made by the reference's own code,
per Gaussian against the float64 oracle, the identity and rigid-motion invariants, and the composite render against
one direct rasterizer call."""
import glob
import math
import os

import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu
GOLD = os.path.join(h.ROOT, "tests", "golden")
MESH_GOLDENS = sorted(os.path.basename(f)[9:-4] for f in glob.glob(os.path.join(GOLD, "editmesh_*.npz"))
                      if "shrot" not in f)


def _cuda(case):
    import torch
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in case.items()}


def _edited(case):
    from sugar_b200 import meshbind
    c = _cuda(case)
    b = meshbind.bind_to_edited_mesh(c["verts"], c["reference_verts"], c["faces"], c["bary"], c["scales_raw"],
                                     c["complex_raw"], c["thickness"])
    return {k: getattr(b, k) for k in ("points", "scaling", "quaternions")}


def _np(d):
    return {k: v.cpu().numpy() for k, v in d.items()}


@pytest.mark.parametrize("name", MESH_GOLDENS)
def test_matches_reference_goldens(name):
    import torch
    g = np.load(os.path.join(GOLD, f"editmesh_{name}.npz"))
    case = {k: torch.from_numpy(g[k]) for k in ("verts", "reference_verts", "faces", "bary", "scales_raw", "complex_raw")}
    case["thickness"] = float(g["thickness"])
    got = _np(_edited(case))
    for k in ("points", "scaling", "quaternions"):
        assert h.rel_err(got[k], g[k]) <= 2e-6, k


def test_large_jittered_soup_matches_fp64_oracle():
    """200k faces, n = 6.  Bound as in tests/test_editmesh_cpu.py: no more than 25 % (+1e-7) farther from float64 than
    the reference's own float32 arithmetic, and 5e-6 at most."""
    import torch
    from oracle import editmesh_oracle as eo
    case = eo.make_case("jitter", F=200_000, n_per=6, seed=11)
    assert max(eo.max_axis_dot(case["verts"], case["faces"]), eo.max_axis_dot(case["reference_verts"], case["faces"])) <= 0.999
    got = _np(_edited(case))
    c = _cuda(case)
    want = {k: v.cpu() for k, v in zip(("points", "scaling", "quaternions"), eo.edited_bind_torch(
        *(c[k].double() if c[k].is_floating_point() else c[k] for k in ("verts", "reference_verts", "faces", "bary",
                                                                         "scales_raw", "complex_raw")), c["thickness"]))}
    ref32 = {k: v.cpu() for k, v in zip(("points", "scaling", "quaternions"), eo.edited_bind_torch(
        c["verts"], c["reference_verts"], c["faces"], c["bary"], c["scales_raw"], c["complex_raw"], c["thickness"]))}
    assert h.rel_err(got["points"], want["points"].numpy()) <= 5e-7
    for k in ("scaling", "quaternions"):
        err, base = h.rel_err(got[k], want[k].numpy()), h.rel_err(ref32[k].numpy(), want[k].numpy())
        assert err <= 5e-6 and err <= 1.25 * base + 1e-7, (k, err, base)
    assert np.abs(np.linalg.norm(got["quaternions"], axis=1) - 1).max() < 1e-5
    assert np.all(got["scaling"][:, 0] == np.float32(case["thickness"]))


@pytest.mark.parametrize("n_per,mesh", [(6, "soup"), (1, "height"), (3, "soup"), (4, "height")])
def test_identity_edit_is_bind_to_mesh(n_per, mesh):
    """At verts == reference_verts every angle change is exactly 0: the frame, the complex number and the quaternion
    are bind_to_mesh's to the bit; the stretch is sum_k b_k * (1 up to rounding)."""
    import torch
    from oracle import editmesh_oracle as eo
    from sugar_b200 import meshbind
    c = _cuda(eo.make_case("identity", F=20_000, n_per=n_per, seed=3, mesh=mesh))
    got = _edited(c)
    with torch.no_grad():
        b = meshbind.bind_to_mesh(c["verts"], c["faces"], c["bary"], c["scales_raw"], c["complex_raw"], c["thickness"])
    assert torch.equal(got["points"], b.points)
    assert torch.equal(got["quaternions"], b.quaternions)
    assert h.rel_err(got["scaling"].cpu().numpy(), b.scaling.cpu().numpy()) <= 1e-6


def _quat_to_matrix(q):
    w, x, y, z = np.moveaxis(q, -1, 0)
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).reshape(q.shape[:-1] + (3, 3))


@pytest.mark.parametrize("mesh,F", [("soup", 20_000), ("height", 800)])
def test_rigid_motion_turns_the_gaussians_with_the_mesh(mesh, F):
    """Scaling unchanged and R(q_new) = Q R(q_old).  The moved vertices are rounded to float32, which by itself tilts a
    face by up to ulp(|v|) / edge: the height field keeps its edges at 1/20 (|v| <= 2 after the motion) so that this
    input rounding stays below the 1e-5 bound; at edge 1/63 it alone reaches 2e-5."""
    import torch
    from oracle import editmesh_oracle as eo
    case = eo.make_case("rigid", F=F, n_per=6, seed=5, mesh=mesh)
    moved = _np(_edited(case))
    rest = _np(_edited(dict(case, verts=case["reference_verts"])))
    Q = eo.rotation([0.3, -0.5, 0.8], 1.1, torch.float64).numpy()         # eo.deform's rigid motion
    assert h.rel_err(moved["scaling"], rest["scaling"]) <= 1e-5
    R_new = _quat_to_matrix(moved["quaternions"].astype(np.float64))
    R_old = _quat_to_matrix(rest["quaternions"].astype(np.float64))
    assert np.abs(R_new - Q @ R_old).max() <= 1e-5


# --- compositor ---

def _scene():
    """Two bound parts (a posed height field, n = 6; a rigidly moved soup, n = 1, rendered through idx) and one plain
    Gaussian set, in front of a camera at z = 4 looking down -z."""
    import torch
    from oracle import editmesh_oracle as eo
    g = torch.Generator().manual_seed(21)
    a = eo.make_case("bent", F=8000, n_per=6, seed=1, mesh="height")
    b = eo.make_case("rigid", F=3000, n_per=1, seed=2)
    for c in (a, b):
        c["scales_raw"] -= 1.5
    b["verts"] = b["verts"] * 0.3
    b["reference_verts"] = b["reference_verts"] * 0.3
    parts, posed = [], []
    for c, idx in ((a, None), (b, torch.randperm(3000, generator=g)[:1700])):
        P = c["scales_raw"].shape[0]
        part = dict(verts=c["reference_verts"], faces=c["faces"], bary=c["bary"], scales_raw=c["scales_raw"],
                    complex_raw=c["complex_raw"], thickness=c["thickness"], densities=torch.randn(P, 1, generator=g),
                    sh=0.5 * torch.randn(P, 16, 3, generator=g))
        if idx is not None:
            part["idx"] = idx
        parts.append(_cuda(part))
        posed.append(c["verts"].cuda())
    Pp = 5000
    q = torch.randn(Pp, 4, generator=g)
    plain = dict(points=(torch.rand(Pp, 3, generator=g) - 0.5) * 2, scaling=torch.rand(Pp, 3, generator=g) * 0.03 + 0.005,
                 quaternions=q / q.norm(dim=1, keepdim=True), opacities=torch.rand(Pp, 1, generator=g),
                 sh=0.5 * torch.randn(Pp, 16, 3, generator=g))
    parts.append(_cuda(plain))
    posed.append(None)
    c2w = torch.eye(4)
    c2w[:3, :3] = torch.tensor(_rot_x(-0.25))        # tilted down toward the parts
    c2w[:3, 3] = torch.tensor([0.2, 1.2, 4.0])
    return parts, posed, c2w


def _rot_x(a):
    return [[1, 0, 0], [0, math.cos(a), -math.sin(a)], [0, math.sin(a), math.cos(a)]]


W, H, FOV = 320, 240, 0.9


def _direct(parts, posed, c2w, colors=None):
    """One rasterizer call on the concatenation of the per-part bind_to_edited_mesh outputs, gathered by idx."""
    import torch
    from sugar_b200 import meshbind, render
    from sugar_b200.diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    cols = {k: [] for k in ("points", "scaling", "quaternions", "opacities", "sh")}
    for part, v in zip(parts, posed):
        if "faces" in part:
            b = meshbind.bind_to_edited_mesh(v, part["verts"], part["faces"], part["bary"], part["scales_raw"],
                                             part["complex_raw"], part["thickness"])
            got = dict(points=b.points, scaling=b.scaling, quaternions=b.quaternions,
                       opacities=torch.sigmoid(part["densities"]), sh=part["sh"])
        else:
            got = {k: part[k] for k in cols}
        for k in cols:
            cols[k].append(got[k] if "idx" not in part else got[k][part["idx"]])
    cat = {k: torch.cat(v) for k, v in cols.items()}
    view, proj, campos = (t.cuda() for t in render.camera_matrices(c2w, FOV, FOV * H / W))
    settings = GaussianRasterizationSettings(H, W, math.tan(FOV * 0.5), math.tan(FOV * H / W * 0.5),
                                             torch.zeros(3, device="cuda"), 1.0, view, proj, 3, campos, False, False)
    kw = dict(shs=cat["sh"]) if colors is None else dict(colors_precomp=colors)
    with torch.no_grad():
        img, _ = GaussianRasterizer(settings)(means3D=cat["points"], means2D=torch.zeros_like(cat["points"]),
                                              opacities=cat["opacities"], scales=cat["scaling"],
                                              rotations=cat["quaternions"], **kw)
    return img.permute(1, 2, 0), cat, campos


def test_composition_render_is_one_direct_rasterizer_call():
    import torch
    from sugar_b200 import compose
    parts, posed, c2w = _scene()
    comp = compose.Composition(parts)
    got = comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed)
    want, _, _ = _direct(parts, posed, c2w)
    assert got.shape == (H, W, 3)
    assert float((want.sum(-1) > 0).float().mean()) > 0.2     # the parts are in view
    assert torch.equal(got, want)
    # a second frame at other vertices rewrites only the bound parts' rows
    got2 = comp.render(c2w, FOV, FOV * H / W, H, W, verts=[None, posed[1], None])
    want2, _, _ = _direct(parts, [parts[0]["verts"], posed[1], None], c2w)
    assert torch.equal(got2, want2)


def test_identity_sh_rotations_are_the_in_kernel_colours():
    import torch
    from sugar_b200 import compose
    parts, posed, c2w = _scene()
    comp = compose.Composition(parts)
    plain = comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed)
    eye = [torch.eye(3)] * 3
    assert torch.equal(comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed, sh_rotations=eye), plain)
    assert torch.equal(comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed, sh_rotations=[None, torch.eye(3), None]),
                       plain)


def test_rotated_sh_colours_in_the_composite():
    """A rotated part's rows take the oracle's rotated colour, the others the plain one, and the image is the direct
    call with those colours."""
    import torch
    from oracle import editmesh_oracle as eo
    from sugar_b200 import compose
    parts, posed, c2w = _scene()
    comp = compose.Composition(parts)
    R = eo.rotation([0.1, 0.9, 0.3], 0.8)
    got = comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed, sh_rotations=[None, R, None])
    _, cat, campos = _direct(parts, posed, c2w)
    s = comp.starts
    rots = [torch.eye(3, dtype=torch.float64), R.double(), torch.eye(3, dtype=torch.float64)]
    want = torch.cat([eo.rotated_colors(cat["points"][s[i]:s[i + 1]].double(), cat["sh"][s[i]:s[i + 1]].double(),
                                        campos.double(), rots[i].cuda(), 3) for i in range(3)])
    assert float((comp.colors - want).abs().max()) <= 1e-5
    img, _, _ = _direct(parts, posed, c2w, colors=comp.colors.clone())
    assert torch.equal(got, img)


@pytest.mark.parametrize("name", ["shrot_deg3", "shrot_deg1"])
def test_rotated_colours_match_reference_goldens(name):
    import torch
    from sugar_b200 import compose
    g = np.load(os.path.join(GOLD, f"editmesh_{name}.npz"))
    t = {k: torch.from_numpy(g[k]).cuda() for k in ("points", "sh", "campos", "rotation")}
    P = t["points"].shape[0]
    # two groups with the same rotation, and the same rows as one group: the group lookup changes nothing
    for starts in ([0, P], [0, P // 3, P]):
        G = len(starts) - 1
        got = compose.sh_colors_rotated(t["points"], t["sh"], t["campos"], torch.tensor(starts).cuda(),
                                        t["rotation"].expand(G, 3, 3).contiguous(), int(g["sh_degree"]))
        assert float((got.cpu() - torch.from_numpy(g["colors"])).abs().max()) <= 1e-5


def test_render_makes_no_host_synchronisation():
    import torch
    from oracle import editmesh_oracle as eo
    from sugar_b200 import compose
    parts, posed, c2w = _scene()
    comp = compose.Composition(parts)
    R = eo.rotation([0.1, 0.9, 0.3], 0.8)
    comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed, sh_rotations=[None, R, None])    # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed)
        comp.render(c2w, FOV, FOV * H / W, H, W, verts=posed, sh_rotations=[None, R, None], bg_color=[0.1, 0.2, 0.3])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_render_rejects_bad_frame_arguments():
    import torch
    from sugar_b200 import compose
    parts, posed, c2w = _scene()
    comp = compose.Composition(parts)
    args = (c2w, FOV, FOV * H / W, H, W)
    with pytest.raises(ValueError, match="verts"):
        comp.render(*args, verts=[posed[0][:-1], None, None])
    with pytest.raises(ValueError, match="not mesh-bound"):
        comp.render(*args, verts=[None, None, posed[0]])
    with pytest.raises(ValueError, match="one entry per part"):
        comp.render(*args, verts=posed[:2])
    with pytest.raises(ValueError, match="forward only"):
        comp.render(*args, verts=[posed[0].clone().requires_grad_(True), None, None])
    with pytest.raises(ValueError, match=r"\[3, 3\]"):
        comp.render(*args, sh_rotations=[None, torch.eye(4), None])
    with pytest.raises(ValueError, match="SH degree"):
        comp.render(*args, sh_deg=4)
