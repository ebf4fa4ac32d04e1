"""The vanilla 3DGS pre-training pieces that need no GPU: train.gs_phase against the vanilla loop's decisions, the
3DGS .ply writer and reader, the SfM point reader, and the vanilla split oracle against SuGaR's."""
import os
import struct
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import densify_oracle as do  # noqa: E402
from oracle import densify_oracle_vanilla as dv  # noqa: E402
from oracle import gs_train_oracle as go  # noqa: E402

train = pytest.importorskip("sugar_b200.train")
from sugar_b200 import gsply, mcubes  # noqa: E402


def test_gs_phase_matches_the_vanilla_loop_at_every_iteration():
    want = go.decisions()
    got = {it: train.gs_phase(it) for it in range(1, 30_001)}
    assert got == want
    assert [it for it in got if "densify" in got[it]] == list(range(600, 15_000, 100))
    assert [it for it in got if got[it].get("size_threshold") == 20] == list(range(3100, 15_000, 100))
    assert [it for it in got if "reset_opacity" in got[it]] == [3000, 6000, 9000, 12000]
    assert [it for it in got if "stats" in got[it]] == list(range(1, 15_000))
    assert [it for it in got if "step" not in got[it]] == [30_000]
    assert [got[it]["sh_degree"] for it in (999, 1000, 1999, 2000, 3000, 29_999)] == [0, 1, 1, 2, 3, 3]


def test_gs_phase_white_background_and_scaled_schedules():
    white = {it: train.gs_phase(it, white_background=True) for it in range(1, 30_001)}
    assert white == go.decisions(white_background=True)
    assert [it for it in white if "reset_opacity" in white[it]] == [500, 3000, 6000, 9000, 12000]
    kw = dict(densify_from_iter=50, densify_until_iter=300, densification_interval=20, opacity_reset_interval=150)
    got = {it: train.gs_phase(it, num_iterations=400, sh_every=100, **kw) for it in range(1, 401)}
    assert got == go.decisions(iterations=400, sh_every=100, **kw)
    assert [it for it in got if "densify" in got[it]] == list(range(60, 300, 20))
    assert [it for it in got if "reset_opacity" in got[it]] == [150]


def test_nerfpp_radius_is_the_float64_restatement():
    c = torch.tensor([[0.1, 0.2, 3.0], [1.0, -0.5, 2.5], [-0.7, 0.9, 2.8], [0.3, 0.3, 0.3]], dtype=torch.float32)
    cd = c.double().numpy()
    want = 1.1 * np.max(np.linalg.norm(cd - cd.mean(0, keepdims=True), axis=1))
    assert mcubes.nerfpp_radius(c) == pytest.approx(want, rel=1e-15)
    assert mcubes.nerfpp_radius(c) == pytest.approx(mcubes.camera_spatial_extent(c), rel=1e-6)


def _raw(P, deg, seed=0):
    g = torch.Generator().manual_seed(seed)
    M = (deg + 1) ** 2
    return dict(points=torch.randn(P, 3, generator=g), sh_dc=torch.randn(P, 1, 3, generator=g),
                sh_rest=torch.randn(P, M - 1, 3, generator=g), densities=torch.randn(P, 1, generator=g),
                scales=torch.randn(P, 3, generator=g) - 3.0, quaternions=torch.randn(P, 4, generator=g))


@pytest.mark.parametrize("deg", [0, 1, 3])
def test_ply_round_trip_is_bit_exact(tmp_path, deg):
    raw = _raw(57, deg, seed=deg)
    path = str(tmp_path / "point_cloud" / "iteration_7000" / "point_cloud.ply")
    gsply.save_gaussians_ply(path, raw)
    back = gsply.load_gaussians_ply(path, sh_degree=deg, device="cpu")
    assert set(back) == set(raw)
    for k in raw:
        assert back[k].shape == raw[k].shape and back[k].dtype == torch.float32, k
        assert torch.equal(back[k].detach().view(torch.int32), raw[k].view(torch.int32)), k
        assert back[k].requires_grad and back[k].is_leaf and back[k].is_contiguous(), k


def _names(deg):
    M = (deg + 1) ** 2
    return (["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] +
            [f"f_rest_{i}" for i in range(3 * (M - 1))] + ["opacity"] + [f"scale_{i}" for i in range(3)] +
            [f"rot_{i}" for i in range(4)])


def test_header_bytes_and_f_rest_order(tmp_path):
    raw = _raw(3, 1, seed=4)
    path = str(tmp_path / "a.ply")
    gsply.save_gaussians_ply(path, raw)
    data = open(path, "rb").read()
    names = _names(1)
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 3\n" +
              "".join(f"property float {n}\n" for n in names) + "end_header\n").encode("ascii")
    assert data.startswith(header) and len(data) == len(header) + 3 * 4 * len(names)
    row1 = np.frombuffer(data[len(header):], dtype="<f4").reshape(3, len(names))[1]
    r = {k: v[1].numpy() for k, v in raw.items()}
    want = np.concatenate([r["points"], np.zeros(3, np.float32), r["sh_dc"][0],
                           # channel-major: all of R's coefficients 1..3, then G's, then B's
                           r["sh_rest"][:, 0], r["sh_rest"][:, 1], r["sh_rest"][:, 2],
                           r["densities"], r["scales"], r["quaternions"]])
    assert np.array_equal(row1.view(np.int32), want.astype(np.float32).view(np.int32))


def _write_ply(path, props, rows, fmt="binary_little_endian", endian="<"):
    """props: [(type, name)]; rows: list of tuples."""
    head = f"ply\nformat {fmt} 1.0\ncomment hand-made\nelement vertex {len(rows)}\n"
    head += "".join(f"property {t} {n}\n" for t, n in props) + "end_header\n"
    code = {"float": "f", "double": "d", "uchar": "B"}
    with open(path, "wb") as f:
        f.write(head.encode("ascii"))
        if fmt == "ascii":
            f.write("".join(" ".join(str(v) for v in r) + "\n" for r in rows).encode("ascii"))
        else:
            for r in rows:
                f.write(struct.pack(endian + "".join(code[t] for t, _ in props), *r))


def test_shuffled_property_order_loads(tmp_path):
    raw = _raw(9, 1, seed=7)
    cols = dict(gsply.gaussian_columns(raw["points"], raw["sh_dc"], raw["sh_rest"], raw["densities"], raw["scales"],
                                       raw["quaternions"]))
    names = list(cols)
    order = [names[i] for i in np.random.default_rng(3).permutation(len(names))]
    # double for positions, float elsewhere: load_ply reads either
    props = [("double" if n in "xyz" else "float", n) for n in order]
    rows = [tuple(float(cols[n][i]) for n in order) for i in range(9)]
    path = str(tmp_path / "shuffled.ply")
    _write_ply(path, props, rows)
    back = gsply.load_gaussians_ply(path, sh_degree=1, device="cpu")
    for k in raw:
        assert torch.equal(back[k].detach(), raw[k]), k


def test_bad_files_are_rejected(tmp_path):
    raw = _raw(4, 3)
    path = str(tmp_path / "deg3.ply")
    gsply.save_gaussians_ply(path, raw)
    with pytest.raises(ValueError, match="f_rest"):
        gsply.load_gaussians_ply(path, sh_degree=2, device="cpu")
    props = [("float", n) for n in _names(0)]
    rows = [tuple(float(i + j) for j in range(len(props))) for i in range(2)]
    for fmt, endian in (("ascii", "<"), ("binary_big_endian", ">")):
        p = str(tmp_path / f"{fmt}.ply")
        _write_ply(p, props, rows, fmt=fmt, endian=endian)
        with pytest.raises(ValueError, match="binary_little_endian"):
            gsply.load_gaussians_ply(p, sh_degree=0, device="cpu")
    p = str(tmp_path / "short.ply")
    _write_ply(p, props, rows)
    with open(p, "r+b") as f:
        f.truncate(os.path.getsize(p) - 1)
    with pytest.raises(ValueError, match="bytes of data"):
        gsply.load_gaussians_ply(p, sh_degree=0, device="cpu")
    p = str(tmp_path / "int.ply")
    _write_ply(p, [("float", "x"), ("int", "y")], [])
    with pytest.raises(ValueError, match="scalar"):
        gsply.read_ply(p)


def test_read_sfm_points_reads_store_ply_layout(tmp_path):
    g = np.random.default_rng(5)
    xyz = g.standard_normal((11, 3)).astype(np.float32)
    rgb = g.integers(0, 256, (11, 3)).astype(np.uint8)
    props = [("float", n) for n in ("x", "y", "z", "nx", "ny", "nz")] + [("uchar", n) for n in ("red", "green", "blue")]
    rows = [tuple(float(v) for v in xyz[i]) + (0.0, 0.0, 0.0) + tuple(int(v) for v in rgb[i]) for i in range(11)]
    path = str(tmp_path / "points3D.ply")
    _write_ply(path, props, rows)
    pts, col = gsply.read_sfm_points(path)
    assert pts.dtype == np.float32 and np.array_equal(pts, xyz)
    assert col.dtype == np.float64 and np.array_equal(col, rgb / 255.0)


def test_vanilla_split_oracle_differs_from_sugar_only_in_r():
    P = 400
    g = torch.Generator().manual_seed(11)
    params = {"points": torch.randn(P, 3, generator=g), "densities": torch.randn(P, 1, generator=g),
              "scales": torch.rand(P, 3, generator=g) * 3.0 - 5.0, "quaternions": torch.randn(P, 4, generator=g) * 2,
              "sh_dc": torch.randn(P, 1, 3, generator=g), "sh_rest": torch.randn(P, 15, 3, generator=g)}
    moments = {k: (torch.rand_like(v), torch.rand_like(v)) for k, v in params.items()}
    stats = {"accum": torch.rand(P, 1, generator=g) * 4e-3, "denom": torch.randint(0, 5, (P, 1), generator=g).float(),
             "max_radii": torch.rand(P, generator=g) * 30}
    args = (2e-4, 0.005, 4.0, 20)
    a = do.densify_and_prune(params, moments, stats, *args, generator=torch.Generator().manual_seed(3))
    b = dv.densify_and_prune(params, moments, stats, *args, generator=torch.Generator().manual_seed(3))
    for k in ("clone", "split", "prune", "samples"):
        assert torch.equal(a[3][k], b[3][k]), k
    S = int(a[3]["split"].sum())
    assert S > 10
    for k in params:
        assert torch.equal(a[1][k][0], b[1][k][0]) and torch.equal(a[1][k][1], b[1][k][1]), k
        if k != "points":
            assert torch.equal(a[0][k], b[0][k]), k
    for k in stats:
        assert torch.equal(a[2][k], b[2][k]), k
    # points: the rows that are not split children agree; the children differ by R only, and both R are rotations of
    # the same unit quaternion, so the children agree to rounding
    pa, pb = a[0]["points"], b[0]["points"]
    same = (pa == pb).all(1)
    assert int((~same).sum()) > 0 and torch.allclose(pa, pb, atol=1e-5, rtol=0)
    n_kept = pa.shape[0] - int((~same).sum())
    assert n_kept >= pa.shape[0] - 2 * S
    q = torch.randn(50, 4, generator=g)
    assert torch.allclose(dv.build_rotation(q), do.quaternion_to_matrix(torch.nn.functional.normalize(q, dim=-1)),
                          atol=1e-6)
