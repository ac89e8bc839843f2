"""The grouped schedule of ts_gemm_kernel<Grouped<Nvfp4Fmt>, N_MMA> on the CPU, for tests.

It is the schedule of tests/grouped_model.py (the same `grouped_schedule`, `group_tile` and `grouped_grid` of
ao_b200/csrc/ts_gemm.cuh) with the token tile chosen from the nvfp4 widths 16 / 32 / 64 / 128 instead of fp8's
16 / 32 / 64, and K in whole 128-k chunks.  The int4 and fp8 weight-only grouped kernels split work the same way;
their tests pass their own format, which sets the ring (streamk_model.ring) of the owners' gather.
"""
import grouped_model as gm


def plan(offs, M, N, K, grid=None, sm=132, fmt="nvfp4"):
    """The grouped split of one launch: grid None = the heuristic, else the forced CTA count."""
    assert fmt in ("nvfp4", "int4", "fp8wo"), fmt
    return gm.plan(offs, M, N, K, grid=grid, sm=sm, fmt=fmt)
