"""Marching cubes in numpy, and the case table it and csrc/sgr_mcubes.cu share.

The table is generated here from one rule rather than typed in:
  * A corner is inside when its value is > level.  Corner (dx, dy, dz) of a cube is bit dx | dy << 1 | dz << 2 of the
    case index.  Edge e = 4 * axis + b joins the two corners that differ in `axis`; b holds the other two coordinates
    in increasing axis order (bit 0 the lower axis).
  * On each of the cube's six faces, walking the face's four corners in a cycle, every run of consecutive inside
    corners is cut off by one segment joining the two crossed edges that bound the run.  On an ambiguous face (inside
    corners on one diagonal only) the two inside corners are therefore separated.  The rule reads only a face's four
    corners, so the two cubes sharing a face draw the same segments there and the surface is watertight.
  * Every crossed edge lies on two faces, so the segments chain into closed loops.  Each loop is oriented so that its
    right-hand (Newell) normal points from the inside corners to the outside ones, i.e. along -grad(density), and
    starts at its smallest edge id.  It is fan-triangulated from its first vertex whose fan diagonals all run through
    the cube's interior: a diagonal between two edges of one face could be drawn by the neighbouring cube as well.

`marching_cubes(volume, level)` applies the table the way the CUDA kernels do and returns the same arrays:
  vertices float64 [V,3] in index space, one per crossed grid edge, ordered by the edge's lower voxel (C order) and
  then by axis x, y, z; vertex = lower corner + t along the axis, t = (level - f1) / (f2 - f1) in double;
  faces int64 [F,3], ordered by cube (C order of its lower corner) and then by table order.

    python oracle/mcubes_oracle.py     # rewrites sugar_b200/csrc/sgr_mcubes_table.h
"""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "sugar_b200", "csrc", "sgr_mcubes_table.h")

CORNERS = np.array([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)])


def _edge(axis, b):
    others = [a for a in range(3) if a != axis]
    lo = [0, 0, 0]
    lo[others[0]] = b & 1
    lo[others[1]] = (b >> 1) & 1
    return tuple(lo)


# EDGE_LO[e]: offset of the edge's lower corner in the cube; EDGE_AXIS[e]: the axis it runs along
EDGE_LO = np.array([_edge(e // 4, e % 4) for e in range(12)])
EDGE_AXIS = np.array([e // 4 for e in range(12)])


def _corner_id(p):
    return int(p[0]) | int(p[1]) << 1 | int(p[2]) << 2


def _edge_id(c0, c1):
    p0, p1 = CORNERS[c0], CORNERS[c1]
    axis = int(np.nonzero(p0 != p1)[0][0])
    lo = np.minimum(p0, p1)
    others = [a for a in range(3) if a != axis]
    return 4 * axis + (int(lo[others[0]]) | int(lo[others[1]]) << 1)


def _face_cycles():
    """The four corners of each cube face in cyclic order."""
    cycles = []
    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in (0, 1):
            ring = []
            for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[axis], p[u], p[v] = side, du, dv
                ring.append(_corner_id(p))
            cycles.append(ring)
    return cycles


FACE_CYCLES = _face_cycles()


def crossed_edges(case):
    ins = [(case >> c) & 1 for c in range(8)]
    return sorted(e for e in range(12)
                  if ins[_corner_id(EDGE_LO[e])] != ins[_corner_id(EDGE_LO[e] + np.eye(3, dtype=int)[EDGE_AXIS[e]])])


def case_loops(case):
    """Oriented edge loops of one case, each starting at its smallest edge id."""
    ins = [(case >> c) & 1 for c in range(8)]
    nbr = {}
    for ring in FACE_CYCLES:
        for i in range(4):
            if ins[ring[i]] or not ins[ring[(i + 1) % 4]]:
                continue
            # a run of inside corners starts at ring[i + 1]; it ends before the next outside corner
            j = (i + 1) % 4
            while ins[ring[(j + 1) % 4]]:
                j = (j + 1) % 4
            a = _edge_id(ring[i], ring[(i + 1) % 4])
            b = _edge_id(ring[j], ring[(j + 1) % 4])
            nbr.setdefault(a, []).append(b)
            nbr.setdefault(b, []).append(a)
    assert all(len(v) == 2 for v in nbr.values()), (case, nbr)
    loops, seen = [], set()
    for start in sorted(nbr):
        if start in seen:
            continue
        loop, prev, cur = [start], None, start
        while True:
            seen.add(cur)
            a, b = nbr[cur]
            nxt = b if a == prev else a
            if nxt == start:
                break
            loop.append(nxt)
            prev, cur = cur, nxt
        loops.append(_orient(loop, ins))
    return loops


def _mid(e):
    return EDGE_LO[e] + 0.5 * np.eye(3)[EDGE_AXIS[e]]


def _outward(e, ins):
    """Unit step along edge e from its inside corner to its outside one."""
    d = np.eye(3)[EDGE_AXIS[e]]
    return d if ins[_corner_id(EDGE_LO[e])] else -d


def _orient(loop, ins):
    pts = [_mid(e) for e in loop]
    n = np.zeros(3)
    for a, b in zip(pts, pts[1:] + pts[:1]):
        n += np.cross(a, b)
    out = sum(_outward(e, ins) for e in loop)
    s = float(n @ out)
    assert abs(s) > 1e-9, loop
    if s < 0:
        loop = loop[::-1]
    k = loop.index(min(loop))
    return loop[k:] + loop[:k]


def _faces_of_edge(e):
    return {i for i, ring in enumerate(FACE_CYCLES)
            if e in {_edge_id(ring[k], ring[(k + 1) % 4]) for k in range(4)}}


def _triangulate(loop):
    """Fan from the first loop vertex (in loop order) whose diagonals all cross the cube's interior.  A diagonal
    joining two edges of one cube face could also be drawn by the cube on the other side of that face, and the
    shared mesh edge would then belong to four triangles."""
    m = len(loop)
    for s in range(m):
        ring = loop[s:] + loop[:s]
        if all(not (_faces_of_edge(ring[0]) & _faces_of_edge(ring[i])) for i in range(2, m - 1)):
            return [(ring[0], ring[i], ring[i + 1]) for i in range(1, m - 1)]
    raise AssertionError(f"no interior fan for loop {loop}")


def build_table():
    """-> (ntri uint8 [256], tris int8 [256, 3 * max_tris] padded with -1)."""
    per_case = []
    for case in range(256):
        tris = []
        for loop in case_loops(case):
            tris.extend(_triangulate(loop))
        per_case.append(tris)
    mx = max(len(t) for t in per_case)
    ntri = np.array([len(t) for t in per_case], np.uint8)
    tab = np.full((256, 3 * mx), -1, np.int8)
    for c, tris in enumerate(per_case):
        if tris:
            tab[c, :3 * len(tris)] = np.array(tris, np.int8).reshape(-1)
    return ntri, tab


def header_text():
    ntri, tab = build_table()
    mx = tab.shape[1] // 3
    out = ["// Generated by oracle/mcubes_oracle.py (python oracle/mcubes_oracle.py); do not edit.",
           "// Marching-cubes case table: corner (dx, dy, dz) is bit dx | dy << 1 | dz << 2 of the case; edge",
           "// 4 * axis + b runs along `axis` from the corner whose other two coordinates are the bits of b (lower axis",
           "// in bit 0).  Triangles are edge triples, oriented with their normal from inside (> level) to outside.",
           "#pragma once",
           f"#define SGR_MC_MAX_TRIS {mx}",
           "__constant__ unsigned char c_mc_ntri[256] = {"]
    for r in range(0, 256, 32):
        out.append("    " + ", ".join(str(int(v)) for v in ntri[r:r + 32]) + ",")
    out.append("};")
    out.append(f"__constant__ signed char c_mc_tris[256][{3 * mx}] = {{")
    for c in range(256):
        out.append("    {" + ", ".join(str(int(v)) for v in tab[c]) + "},")
    out.append("};")
    return "\n".join(out) + "\n"


_TABLE = None


def table():
    global _TABLE
    if _TABLE is None:
        _TABLE = build_table()
    return _TABLE


def marching_cubes(volume, level):
    """The CUDA kernels' marching cubes in numpy: -> (vertices float64 [V,3], faces int64 [F,3])."""
    f = np.asarray(volume, np.float32).astype(np.float64)
    level = float(level)
    ins = f > level
    R = f.shape
    cross = np.zeros(R + (3,), bool)
    cross[:-1, :, :, 0] = ins[:-1] != ins[1:]
    cross[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    cross[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    ids = (np.cumsum(cross.reshape(-1)) - 1).reshape(cross.shape)
    vox, axis = np.nonzero(cross.reshape(-1, 3))
    ijk = np.stack(np.unravel_index(vox, R), 1)
    f1 = f[tuple(ijk.T)]
    f2 = f[tuple((ijk + np.eye(3, dtype=np.int64)[axis]).T)]
    t = (level - f1) / (f2 - f1)
    verts = ijk.astype(np.float64)
    verts[np.arange(len(vox)), axis] += t
    if min(R) < 2:
        return verts, np.zeros((0, 3), np.int64)
    ntri, tab = table()
    C = tuple(n - 1 for n in R)
    case = np.zeros(C, np.int64)
    for c in range(8):
        dx, dy, dz = CORNERS[c]
        case |= ins[dx:dx + C[0], dy:dy + C[1], dz:dz + C[2]].astype(np.int64) << c
    cubes = np.nonzero(ntri[case.reshape(-1)])[0]
    cc = case.reshape(-1)[cubes]
    cijk = np.stack(np.unravel_index(cubes, C), 1)
    mx = tab.shape[1] // 3
    faces = np.full((len(cubes), mx, 3), -1, np.int64)
    for s in range(mx):
        live = ntri[cc] > s
        for k in range(3):
            e = tab[cc[live], 3 * s + k].astype(np.int64)
            p = cijk[live] + EDGE_LO[e]
            faces[live, s, k] = ids[p[:, 0], p[:, 1], p[:, 2], EDGE_AXIS[e]]
    faces = faces.reshape(-1, 3)
    return verts, faces[faces[:, 0] >= 0]


def euler_characteristic(n_verts, faces):
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), 1)
    return n_verts - len(np.unique(e, axis=0)) + len(faces)


def directed_edge_counts(faces):
    """-> (counts of each undirected edge, whether every directed edge occurs at most once)."""
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    _, dc = np.unique(d, axis=0, return_counts=True)
    _, uc = np.unique(np.sort(d, 1), axis=0, return_counts=True)
    return uc, bool((dc == 1).all())


def mesh_area(verts, faces):
    v = np.asarray(verts, np.float64)
    return 0.5 * np.linalg.norm(np.cross(v[faces[:, 1]] - v[faces[:, 0]], v[faces[:, 2]] - v[faces[:, 0]]), axis=1).sum()


if __name__ == "__main__":
    with open(HEADER, "w") as fh:
        fh.write(header_text())
    print(HEADER, "max triangles per case:", table()[1].shape[1] // 3)
