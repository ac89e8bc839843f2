"""A CPU restatement of the grouped schedule of ts_gemm_kernel<Grouped<Fmt>, N_MMA> (torch._grouped_mm), for tests.

It mirrors `grouped_schedule`, `group_tile` and `grouped_grid` of ao_b200/csrc/ts_gemm.cuh and the upper-bound grid of
`launch_gemm<..., GROUPED>`; the walk of each CTA is streamk_model.walk.  Keep the two in step: a change to the grouped
schedule there needs the same change here, or test_grouped_schedule.py checks a schedule the kernel does not run.
"""
from dataclasses import dataclass, field

import streamk_model as sk

MAX_EXPERTS = 1024
MIN_UNITS = 4


def cumulative(rows):
    """offs of torch._grouped_mm from the rows of each expert: the cumulative row ends."""
    out, s = [], 0
    for r in rows:
        s += r
        out.append(s)
    return out


def row_ends(offs, M):
    """end[e] = min(M, max(0, offs[0..e])): every offs[e] clamped into [end[e-1], M]."""
    ends, run = [], 0
    for o in offs:
        run = max(run, o)
        ends.append(min(run, M))
    return ends


def mblock_prefix(ends, width):
    mbp, start = [0], 0
    for e in ends:
        mbp.append(mbp[-1] + -(-(e - start) // width))
        start = e
    return mbp


def group_tile(ends, mbp, j, width):
    """(expert, first row, expert's end row) of (expert, m-block) pair j: the largest e with mbp[e] <= j."""
    lo, hi = 0, len(ends) - 1
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if mbp[mid] <= j:
            lo = mid
        else:
            hi = mid - 1
    start = ends[lo - 1] if lo > 0 else 0
    return lo, start + (j - mbp[lo]) * width, ends[lo]


def host_grid(M, E, n_tiles, KT, width, forced=0, sm=132):
    """launch_gemm<..., GROUPED>: the grid for the upper bound n_tiles * (ceil(M / width) + min(E, M)) * KT."""
    units = n_tiles * (-(-M // width) + min(E, M)) * KT
    if forced:
        return units, max(1, min(forced, sm, units))
    return units, sk.default_grid(units, sm, MIN_UNITS)


def grouped_grid(G, U, forced):
    if U == 0:
        return 0
    cap = U if forced else max(1, U // MIN_UNITS)
    return min(cap, G)


@dataclass
class GroupedPlan:
    M: int
    N: int
    K: int
    E: int
    width: int
    n_tiles: int
    KT: int
    ends: list
    mbp: list
    U: int
    U_bound: int
    G_host: int
    G: int
    fmt: str = "fp8"
    ctas: list = field(default_factory=list)     # ctas[b] = list of streamk_model.Seg (b < G)
    owners: dict = field(default_factory=dict)   # split tile -> (owner CTA, [contributor CTAs])

    def tile(self, t):
        """(expert, first row, end row, n-tile) of tile t."""
        e, row0, row_end = group_tile(self.ends, self.mbp, t // self.n_tiles, self.width)
        return e, row0, row_end, t % self.n_tiles

    def contributor_counts(self):
        return [len(c) for _, c in self.owners.values()]

    def gather_split(self, c):
        return sk.gather_split(self.fmt, self.width, True, c)

    def owner_cols(self, t):
        """Valid token columns of tile t: the rows of its expert from its first row on, at most the width."""
        _, row0, row_end, _ = self.tile(t)
        return min(row_end - row0, self.width)


def plan(offs, M, N, K, grid=None, sm=132, fmt="fp8"):
    """The grouped split of one launch of Grouped<fmt>: grid None = the heuristic, else the forced CTA count."""
    E = len(offs)
    width = sk.n_mma(fmt, M)
    KT = sk.k_chunks(fmt, K)
    n_tiles = -(-N // sk.ROWS)
    ends = row_ends(offs, M)
    mbp = mblock_prefix(ends, width)
    U = n_tiles * mbp[-1] * KT
    U_bound, G_host = host_grid(M, E, n_tiles, KT, width, grid or 0, sm)
    G = grouped_grid(G_host, U, bool(grid))
    p = GroupedPlan(M, N, K, E, width, n_tiles, KT, ends, mbp, U, U_bound, G_host, G, fmt)
    for b in range(G):
        u0, u1 = sk.unit_begin(b, U, G), sk.unit_begin(b + 1, U, G)
        p.ctas.append(sk.walk(u0, u1 - u0, KT) if u1 > u0 else [])
    for b, segs in enumerate(p.ctas):
        if segs and segs[-1].kind == sk.OWNER:
            t = segs[-1].tile
            p.owners[t] = (b, list(range(b + 1, sk.cta_of_unit(t * KT + KT - 1, U, G) + 1)))
    return p
