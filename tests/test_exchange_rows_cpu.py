"""CPU side of tests/test_gpu_exchange_rows.py: the peer reduce's 16-byte unit partition restated, and the row checks of
the GPU file shown to catch what the per-tensor |a - b|_inf / |b|_inf <= 1e-4 of test_gpu_parallel.py lets through."""
import ctypes

import numpy as np
import pytest

import helpers as h
import test_gpu_exchange_rows as ex

UNITS_PER_BLOCK = 64 * 11 // 4     # one 64-record block of 44-byte records = 176 16-byte units


def owned_units(p0, p1, N, r):
    """Units [q0, q1) of the chunk [p0, p1) that rank r of N sums: sgr_peer_reduce_records_synced (sgr_peer.cu)."""
    nb = (p1 - p0 + 63) // 64
    bs, be = (nb * r + N - 1) // N, (nb * (r + 1) + N - 1) // N
    Q0, Qend = p0 * 11 // 4, (p1 * 11 + 3) // 4
    q1 = min(Q0 + be * UNITS_PER_BLOCK, Qend)
    return min(Q0 + bs * UNITS_PER_BLOCK, q1), q1


def producer(i, p0, p1, N):
    """Rank whose staging array receives record i of the chunk [p0, p1): CTA b of nb sends to b * N / nb
    (sgr_backward.cu, PreBwdArgs::stage_tab)."""
    nb = (p1 - p0 + 63) // 64
    return (i - p0) // 64 * N // nb


def chunk_ranges(P, chunks, taper):
    """The [p0, p1) of every chunk the per-Gaussian pass runs (and hands to the reduce), from the library."""
    from sugar_b200 import _lib
    p0, p1 = ctypes.c_int32(), ctypes.c_int32()
    n = min(chunks, (P + 63) // 64)          # backward_chunks(): at most one chunk per CTA
    out = []
    for c in range(n):
        assert _lib.lib.sgr_backward_chunk_range(P, chunks, c, int(taper), ctypes.byref(p0), ctypes.byref(p1)) == 0
        out.append((p0.value, p1.value))
    return out


def check_partition(P, p0, p1, N, per_unit):
    Q0, Qend = p0 * 11 // 4, (p1 * 11 + 3) // 4
    assert p0 % 64 == 0 and Q0 * 4 == p0 * 11
    at = Q0
    for r in range(N):
        q0, q1 = owned_units(p0, p1, N, r)
        assert q0 == at and q0 <= q1, (P, p0, p1, N, r, q0, q1, at)     # no gap, no overlap, in rank order
        at = q1
        if q1 == q0:
            continue
        # a unit's floats [4q, 4q + 4): those inside the chunk belong to records rank r produced, the rest is the
        # padding behind the last record of the whole array (never another chunk's records)
        assert 4 * q1 <= 11 * p1 or p1 == P, (P, p0, p1, N, r)
        if per_unit:
            q = np.arange(q0, q1)
            first, last = 4 * q // 11, np.minimum(4 * q + 3, 11 * p1 - 1) // 11
            for rec in (first, last):
                assert np.all((rec - p0) // 64 * N // ((p1 - p0 + 63) // 64) == r), (P, p0, p1, N, r)
        else:   # producers are non-decreasing in the record index: the slice's two ends decide
            a, b = 4 * q0 // 11, min(4 * q1 - 1, 11 * p1 - 1) // 11
            assert producer(a, p0, p1, N) == r and producer(b, p0, p1, N) == r, (P, p0, p1, N, r)
    assert at == Qend, (P, p0, p1, N, at, Qend)


@pytest.mark.parametrize("P", [1, 63, 64, 65, 6001, 3_000_000])
def test_reduce_units_partition_every_chunk(P):
    """For every chunk range the library hands out (1-16 chunks, taper on and off) and 1-64 ranks: the ranks' unit
    slices tile [11 p0 / 4, ceil(11 p1 / 4)) in rank order, and every unit goes to the rank whose per-Gaussian pass
    produced its records; the chunks tile [0, P)."""
    per_unit = P <= 6001
    for chunks in range(1, 17):
        for taper in (False, True):
            ranges = chunk_ranges(P, chunks, taper)
            assert ranges[0][0] == 0 and ranges[-1][1] == P
            assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
            for p0, p1 in ranges:
                for N in range(1, 65):
                    check_partition(P, p0, p1, N, per_unit)


def test_tail_chunks_leave_ranks_without_units():
    """The case the GPU file's 16 tapered chunks at P = 6001 rely on: chunks with fewer blocks than ranks (and empty
    ones), where a rank owns no unit and its reduce kernel only runs the flag handshake."""
    ranges = chunk_ranges(6001, 16, True)
    nbs = [(p1 - p0 + 63) // 64 for p0, p1 in ranges]
    assert 0 in nbs and 1 in nbs
    for N, me in ((3, 1), (5, 4), (16, 9)):
        idle = [c for c, (p0, p1) in enumerate(ranges) if owned_units(p0, p1, N, me)[0] == owned_units(p0, p1, N, me)[1]
                and p1 > p0]
        assert idle, (N, me)


# ---------------------------------------------------------------------------------------------------------------------
# the row checks against the per-tensor check, on synthetic arrays
def _records(P, seed):
    return ex.synthetic_records(P, seed)


def test_sums_check_catches_a_unit_left_out():
    P = 1000
    stages = [_records(P, s).reshape(-1) for s in range(3)]
    S = ex.reduce_in_rank_order(stages)
    ex.check_sums("intact", [S, S.copy()], stages)
    mag = np.abs(S).reshape(-1, 4).max(1)
    q = int(np.flatnonzero(mag < 1e-5 * np.abs(S).max())[len(mag) // 10 % 7])   # a small unit inside a slice
    bad = S.copy()
    bad[4 * q:4 * q + 4] = 0.0                                                   # never stored: the array's old zeros
    assert h.rel_err(bad, S) <= 1e-4
    with pytest.raises(pytest.fail.Exception, match=f"unit {q}"):
        ex.check_sums("unit left out", [S, bad], stages)


def _dsh_scene(P, nviews, seed=41):
    from sugar_b200 import scenes
    base = scenes.make_scene(P, 160, 96, seed=seed, camera="posed")
    campos = [ex.view_scene(base, j).campos for j in range(nviews)]
    return base.means3D, campos


def _rounded(ref, M):
    return ref[:, :M].astype(np.float32)


def test_dsh_check_catches_a_view_summed_twice():
    P, V, deg, scale = 2000, 3, 3, 1.0 / 3
    means, campos = _dsh_scene(P, V)
    f = ex.synthetic_factors(P, V, seed=3)
    # view 2 is a far view: it sees a tenth of the Gaussians, weakly, and some of them no other view sees
    f[2] *= 1e-6
    f[2, np.arange(P) % 10 != 3] = 0
    f[:2, np.arange(P) % 30 == 3] = 0
    ref, wt = ex.dsh_reference(means, campos, f, deg, scale)
    assert ex.check_dsh("intact", _rounded(ref, 16), ref, wt, deg) <= 0.5
    twice = ref + ex.dsh_reference(means, [campos[2]], [f[2]], deg, scale)[0]
    assert h.rel_err(_rounded(twice, 16), ref) <= 1e-4
    with pytest.raises(pytest.fail.Exception, match="dL_dsh of Gaussian"):
        ex.check_dsh("view 2 twice", _rounded(twice, 16), ref, wt, deg)


@pytest.mark.parametrize("level", [1e-3, 1e-5])
def test_row_checks_catch_a_zeroed_row(level):
    """A Gaussian whose gradient row is `level` x the tensor's largest entry, zeroed: the split's bit-for-bit check and
    the dL_dsh bound fail.  Per tensor, 1e-5 passes |a - b|_inf / |b|_inf <= 1e-4 (1e-3 does not)."""
    P, scale, deg = 2000, 0.3, 3
    rec = _records(P, 7)
    rows = np.abs(rec).max(1)
    g = int(np.argmin(np.abs(rows / rows.max() - level)))
    rec[g] *= np.float32(level * rows.max() / rows[g])
    out = {k: (rec[:, a:b] * np.float32(scale)) for k, (a, b) in ex.SPLIT.items()}
    ex.check_split("intact", out, rec, scale)
    k = max(ex.SPLIT, key=lambda k: np.abs(rec[g, ex.SPLIT[k][0]:ex.SPLIT[k][1]]).max())
    out[k] = out[k].copy()
    out[k][g] = 0
    per_tensor = h.rel_err(np.concatenate([out[n] for n in ex.SPLIT], 1), rec * np.float32(scale))
    assert (per_tensor <= 1e-4) == (level < 1e-4), per_tensor
    with pytest.raises(AssertionError, match=f"row {g}"):
        ex.check_split("zeroed row", out, rec, scale)

    means, campos = _dsh_scene(P, 2)
    f = ex.synthetic_factors(P, 2, seed=5)
    ref, _ = ex.dsh_reference(means, campos, f, deg, scale)
    mag = np.abs(ref).max((1, 2))
    g = int(np.argsort(mag)[P // 2])                       # a Gaussian both views see, scaled to `level` of the largest
    f[:, g] *= np.float32(level * mag.max() / mag[g])
    ref, wt = ex.dsh_reference(means, campos, f, deg, scale)
    got = _rounded(ref, 16)
    got[g] = 0
    per_tensor = h.rel_err(got, ref)
    assert (per_tensor <= 1e-4) == (level < 1e-4), per_tensor
    with pytest.raises(pytest.fail.Exception, match=f"Gaussian {g} "):
        ex.check_dsh("zeroed row", got, ref, wt, deg)
