"""Deterministic synthetic Gaussian clouds + cameras (SURVEY.md section 8d).

There is no dataset or checkpoint access, so tests and bench.py render seeded synthetic
clouds of the Gaussian count / resolution / SH degree BASELINE.json names.  Everything is
generated on the CPU with numpy's PCG64 so that the CPU oracle, the committed golden
fixtures and the GPU runs all see bit-identical inputs.

Camera conventions follow the reference's callers (sugar_scene/sugar_model.py:2126-2161,
sugar_utils/graphics_utils.py:38-85): `viewmatrix` is the world->view matrix TRANSPOSED
(row-vector convention), `projmatrix = viewmatrix @ P^T`; the kernels read both column-major.
"""
import math
from typing import NamedTuple, Optional

import numpy as np


class Scene(NamedTuple):
    means3D: np.ndarray        # [P,3]
    scales: np.ndarray         # [P,3]  (already activated: exp)
    rotations: np.ndarray      # [P,4]  (w,x,y,z), normalised
    opacities: np.ndarray      # [P,1]  (already activated: sigmoid)
    shs: np.ndarray            # [P,16,3]
    colors_precomp: np.ndarray  # [P,3] in [0,1]
    viewmatrix: np.ndarray     # [4,4] transposed world->view
    projmatrix: np.ndarray     # [4,4] full projection, transposed
    campos: np.ndarray         # [3]
    tanfovx: float
    tanfovy: float
    width: int
    height: int


def projection_matrix(znear: float, zfar: float, tanfovx: float, tanfovy: float) -> np.ndarray:
    """getProjectionMatrix (sugar_utils/graphics_utils.py:65-85), untransposed."""
    top = tanfovy * znear
    right = tanfovx * znear
    Pm = np.zeros((4, 4), np.float64)
    Pm[0, 0] = 2.0 * znear / (2 * right)
    Pm[1, 1] = 2.0 * znear / (2 * top)
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    return Pm


def _rot(axis: np.ndarray, angle: float) -> np.ndarray:
    axis = axis / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * (K @ K)


def make_scene(P: int, width: int, height: int, seed: int = 0, fov_x_deg: float = 60.0,
               camera: str = "identity", px_sigma: float = 1.5, mesh_bound: bool = False,
               frac_behind: float = 0.02, lateral: float = 1.1,
               zrange=(2.0, 10.0)) -> Scene:
    """Cloud of P Gaussians in front of a pinhole camera.

    z ~ U[zrange]; x,y ~ z*tanfov*U[-lateral,lateral] (about 17% outside the frustum laterally
    for lateral=1.1); `frac_behind` of the points get z in [-1,0.2] to exercise the near cull;
    log-normal scales giving ~`px_sigma` pixels at mid depth; `mesh_bound` flattens the first
    axis (refine.py-style surface-aligned Gaussians, sugar_model.py:438-441).
    camera="identity": world == camera.  camera="posed": a seeded rigid transform.
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    tanfovx = math.tan(math.radians(fov_x_deg) / 2)
    tanfovy = tanfovx * height / width
    focal_x = width / (2 * tanfovx)
    z = rng.uniform(zrange[0], zrange[1], P)
    nb = int(round(frac_behind * P))
    if nb:
        z[rng.choice(P, nb, replace=False)] = rng.uniform(-1.0, 0.2, nb)
    zz = np.where(np.abs(z) < 0.3, 0.3, np.abs(z))
    x = zz * tanfovx * rng.uniform(-lateral, lateral, P)
    y = zz * tanfovy * rng.uniform(-lateral, lateral, P)
    cam_pts = np.stack([x, y, z], 1)
    zmid = 0.5 * (zrange[0] + zrange[1])
    s0 = zmid * px_sigma / focal_x
    scales = np.exp(rng.normal(math.log(s0), 0.5, (P, 3)))
    if mesh_bound:
        scales[:, 0] = 1e-6 * (zrange[1] - zrange[0])
    q = rng.normal(size=(P, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    opac = 1.0 / (1.0 + np.exp(-rng.normal(0.0, 2.0, (P, 1))))
    shs = np.concatenate([rng.normal(0, 0.5, (P, 1, 3)), rng.normal(0, 0.1, (P, 15, 3))], 1)
    colors = rng.uniform(0, 1, (P, 3))

    if camera == "identity":
        Rwc = np.eye(3)
        twc = np.zeros(3)
    else:
        Rwc = _rot(rng.normal(size=3), rng.uniform(0.3, 2.5))   # world->cam rotation
        twc = rng.normal(size=3) * 2.0
    # x_cam = Rwc x_world + twc  ->  x_world = Rwc^T (x_cam - twc)
    world = (cam_pts - twc) @ Rwc
    V = np.eye(4)
    V[:3, :3] = Rwc
    V[:3, 3] = twc
    Pm = projection_matrix(0.01, 100.0, tanfovx, tanfovy)
    viewmatrix = V.T.astype(np.float32)
    projmatrix = (V.T @ Pm.T).astype(np.float32)
    campos = (-Rwc.T @ twc).astype(np.float32)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return Scene(f32(world), f32(scales), f32(q), f32(opac), f32(shs), f32(colors), viewmatrix, projmatrix,
                 campos, float(np.float32(tanfovx)), float(np.float32(tanfovy)), width, height)


def with_camera_offset(sc: Scene, yaw: float, shift) -> Scene:
    """The same cloud seen from a camera moved relative to `sc`'s: x_cam' = R_y(yaw) x_cam + shift."""
    V = sc.viewmatrix.astype(np.float64).T
    D = np.eye(4)
    D[:3, :3] = _rot(np.array([0.0, 1.0, 0.0]), yaw)
    D[:3, 3] = np.asarray(shift, np.float64)
    V2 = D @ V
    Pm = projection_matrix(0.01, 100.0, sc.tanfovx, sc.tanfovy)
    campos = (-V2[:3, :3].T @ V2[:3, 3]).astype(np.float32)
    return sc._replace(viewmatrix=V2.T.astype(np.float32), projmatrix=(V2.T @ Pm.T).astype(np.float32), campos=campos)


def height_field_mesh(nx: int, ny: int, seed: int = 0, amplitude: float = 0.05, noise: float = 0.01,
                      permute: bool = False):
    """Connected triangle mesh of a noisy height field over the unit square: an nx x ny vertex grid, two triangles
    per cell (F = 2 (nx - 1)(ny - 1)), z = amplitude * (a few smooth waves) + noise * grid spacing * N(0, 1), so
    that adjacent faces are a few hundredths of a radian apart, as on the smooth meshes refinement binds to.
    `permute` shuffles the vertex ids and the face order (seeded), for the scattered access of a decimated Poisson
    mesh.  -> (verts float32 [V,3], faces int64 [F,3])."""
    rng = np.random.Generator(np.random.PCG64(seed))
    x, y = np.meshgrid(np.linspace(0.0, 1.0, nx), np.linspace(0.0, 1.0, ny), indexing="xy")
    h = 1.0 / max(nx - 1, ny - 1, 1)
    z = amplitude * (np.sin(2 * math.pi * (1.5 * x + 0.3)) * np.cos(2 * math.pi * (1.0 * y - 0.2)) + 0.5 * x * y)
    z = z + noise * h * rng.normal(size=z.shape)
    verts = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    i, j = np.meshgrid(np.arange(nx - 1), np.arange(ny - 1), indexing="xy")
    v00 = (j * nx + i).ravel()
    v10, v01, v11 = v00 + 1, v00 + nx, v00 + nx + 1
    faces = np.stack([np.stack([v00, v10, v11], 1), np.stack([v00, v11, v01], 1)], 1).reshape(-1, 3)
    if permute:
        perm = rng.permutation(len(verts))            # new id of old vertex k is inv[k]
        inv = np.empty_like(perm)
        inv[perm] = np.arange(len(perm))
        verts = verts[perm]
        faces = inv[faces][rng.permutation(len(faces))]
    return np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(faces, np.int64)


def icosphere(subdivisions: int, radius: float = 1.0):
    """Closed subdivided icosahedron (every edge shared by exactly two faces): V = 10 * 4^s + 2, F = 20 * 4^s,
    outward winding.  -> (verts float32 [V,3], faces int64 [F,3])."""
    t = (1.0 + math.sqrt(5.0)) / 2.0
    verts = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                      [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    faces = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                      [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
                      [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], np.int64)
    verts /= np.linalg.norm(verts, axis=1, keepdims=True)
    for _ in range(subdivisions):
        edges = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
        uniq, inv = np.unique(edges, axis=0, return_inverse=True)
        mid = verts[uniq[:, 0]] + verts[uniq[:, 1]]
        verts = np.concatenate([verts, mid / np.linalg.norm(mid, axis=1, keepdims=True)])
        m = len(verts) - len(uniq) + inv.reshape(3, -1).T   # midpoints of (v0 v1), (v1 v2), (v2 v0)
        a, b, c = faces.T
        faces = np.concatenate([np.stack([a, m[:, 0], m[:, 2]], 1), np.stack([b, m[:, 1], m[:, 0]], 1),
                                np.stack([c, m[:, 2], m[:, 1]], 1), m])
    return np.ascontiguousarray(verts * radius, np.float32), np.ascontiguousarray(faces, np.int64)


def upstream_grad(width: int, height: int, seed: int = 1) -> np.ndarray:
    """Fixed dL/dimage: loss = (image * Wt).sum(), Wt ~ N(0,1)/(3HW)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return (rng.normal(size=(3, height, width)) / (3.0 * height * width)).astype(np.float32)
