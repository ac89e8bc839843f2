"""The grouped schedule of ts_gemm_kernel<Grouped<Nvfp4Fmt>, N_MMA> on the CPU, for tests.

It is the schedule of tests/grouped_model.py (the same `grouped_schedule`, `group_tile` and `grouped_grid` of
ao_b200/csrc/ts_gemm.cuh) with the token tile chosen from the nvfp4 widths 16 / 32 / 64 / 128 instead of fp8's
16 / 32 / 64, and K in whole 128-k chunks.
"""
import grouped_model as gm
import streamk_model as sk


def plan(offs, M, N, K, grid=None, sm=132):
    """The grouped split of one nvfp4 launch: grid None = the heuristic, else the forced CTA count."""
    E = len(offs)
    width = sk.n_mma("nvfp4", M)
    KT = sk.k_chunks("nvfp4", K)
    n_tiles = -(-N // sk.ROWS)
    ends = gm.row_ends(offs, M)
    mbp = gm.mblock_prefix(ends, width)
    U = n_tiles * mbp[-1] * KT
    U_bound, G_host = gm.host_grid(M, E, n_tiles, KT, width, grid or 0, sm)
    G = gm.grouped_grid(G_host, U, bool(grid))
    p = gm.GroupedPlan(M, N, K, E, width, n_tiles, KT, ends, mbp, U, U_bound, G_host, G)
    for b in range(G):
        u0, u1 = sk.unit_begin(b, U, G), sk.unit_begin(b + 1, U, G)
        p.ctas.append(sk.walk(u0, u1 - u0, KT) if u1 > u0 else [])
    for b, segs in enumerate(p.ctas):
        if segs and segs[-1].kind == sk.OWNER:
            t = segs[-1].tile
            p.owners[t] = (b, list(range(b + 1, sk.cta_of_unit(t * KT + KT - 1, U, G) + 1)))
    return p
