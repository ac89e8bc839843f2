"""CPU checks of the grouped schedule of the fp8 grouped GEMM (tests/grouped_model.py, a restatement of
ao_b200/csrc/ts_gemm.cuh), for seeded random and adversarial offs:

* every row in [0, end) (end = offs[-1] clamped into [0, M]) is computed by exactly one (expert, m-block) per n-tile,
  and each by its own expert;
* no tile reads an activation row, a weight row or a weight scale outside its tensor, and none writes outside [0, M);
* the device-side grid never exceeds U or the launched grid, every CTA below it has units, and every owner's
  contributors hold the tile as their first (CONTRIB) segment;
* the forced grids of tests/test_grouped_mm_gpu.py reach CONTRIB, FULL and OWNER segments.
"""
import random

import pytest

import grouped_model as gm
import streamk_model as sk


def _offs_cases():
    rng = random.Random(1234)
    cases = []
    for _ in range(60):   # seeded random routings, some rows past offs[-1]
        E = rng.choice([1, 2, 3, 8, 16, 64, 128])
        rows = [rng.choice([0, 0, 1, 2, 5, 16, 17, 40, 64, 65, 130]) for _ in range(E)]
        M = max(1, sum(rows) + rng.choice([0, 0, 3]))
        cases.append((list(_cum(rows)), M))
    cases += [
        ([0, 0, 0, 0], 7),                   # every expert empty: no units, no CTA
        ([0, 0, 37, 37], 37),                # one expert with every row
        ([200], 200), ([1], 1), ([64], 64), ([65], 65),
        ([3, 3, 10], 30),                    # offs[-1] < M
        ([9, 4, -3, 30, 12, 500], 40),       # decreasing, negative, past M
        ([-5, -1, 0, 3], 8),
        ([100, 200], 64),
        ([-1], 5),
        (list(range(0, 1024)), 1023),        # E = 1024, the table's cap: one row per expert
        ([2**31 - 1] * 3, 17),
    ]
    return cases


def _cum(rows):
    s = 0
    for r in rows:
        s += r
        yield s


SHAPES = [(256, 1024), (144, 512), (640, 1024), (128, 16384)]


def _check(offs, M, N, K, grid, sm=132):
    p = gm.plan(offs, M, N, K, grid=grid, sm=sm)
    E = len(offs)
    end = p.ends[-1]
    assert 0 <= end <= M
    assert p.G <= p.G_host and p.U <= p.U_bound and p.G <= max(p.U, 0)
    if p.U == 0:
        assert p.G == 0 and end == 0
        return p
    assert p.G >= 1
    covered = [[0] * p.n_tiles for _ in range(end)]
    for t in range(p.U // p.KT):
        e, row0, row_end, n_tile = p.tile(t)
        assert 0 <= e < E and 0 <= row0 < row_end <= M, (offs, M, t, e, row0, row_end)
        start = p.ends[e - 1] if e > 0 else 0
        assert start <= row0 < p.ends[e] == row_end
        # weight rows e*N + 128*n_tile ..: the box starts inside the [E*N, K] map; features past N are never stored
        assert 0 <= e * N + n_tile * sk.ROWS < E * N
        for m in range(row0, min(row0 + p.width, row_end)):
            covered[m][n_tile] += 1
    assert all(c == [1] * p.n_tiles for c in covered), f"rows not covered once: offs={offs} M={M}"
    owned = [0] * p.U
    for b, segs in enumerate(p.ctas):
        assert segs, f"CTA {b} of the device grid {p.G} has no units"
        for s in segs:
            for u in range(s.tile * p.KT + s.kc0, s.tile * p.KT + s.kc0 + s.count):
                owned[u] += 1
                assert sk.cta_of_unit(u, p.U, p.G) == b
    assert owned == [1] * p.U
    for t, (owner, contribs) in p.owners.items():
        for c in contribs:
            assert c < p.G and p.ctas[c] and p.ctas[c][0].tile == t and p.ctas[c][0].kind == sk.CONTRIB
    return p


@pytest.mark.parametrize("N,K", SHAPES)
def test_schedule_invariants(N, K):
    for offs, M in _offs_cases():
        grids = {None, 1, 2, 3, 7, 64, 131, 132, 500}
        for G in grids:
            _check(offs, M, N, K, G)


def test_row_ends_clamp():
    assert gm.row_ends([9, 4, -3, 30, 12, 500], 40) == [9, 9, 9, 30, 30, 40]
    assert gm.row_ends([-5, -1, 0, 3], 8) == [0, 0, 0, 3]
    assert gm.mblock_prefix([9, 9, 9, 30, 30, 40], 16) == [0, 1, 1, 1, 3, 3, 4]


def test_gpu_cases_reach_every_segment_kind():
    import test_grouped_mm_gpu as suite

    kinds = set()
    widths = set()
    for rows, N, K, tail, grids in suite.GROUPED_CASES:
        offs, M = list(_cum(rows)), sum(rows) + tail
        for G in [None] + suite.grids_of(rows, N, K, tail, grids, 132):
            p = _check(offs, M, N, K, G)
            widths.add(p.width)
            for segs in p.ctas:
                kinds.update(s.kind for s in segs)
                if [s.kind for s in segs][:1] == [sk.CONTRIB] and segs[-1].kind == sk.OWNER and len(segs) > 2:
                    kinds.add("contrib_full_owner")
    assert {sk.FULL, sk.CONTRIB, sk.OWNER, "contrib_full_owner"} <= kinds, kinds
    assert widths == {16, 32, 64}, widths
