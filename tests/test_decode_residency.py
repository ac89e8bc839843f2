"""Two decode CTAs fit on one SM, so that the next linear's CTA becomes resident beside the running one (PDL).

The decode instantiations of ts_gemm_kernel (N_MMA 16 and 32) of the formats with Fmt::DECODE_2CTA must launch with
at most 80 registers per thread (65536 / (2 x 384), rounded down to the allocation granule of 8), and their shared
memory (ts_gemm.cuh Cfg::SMEM_BYTES, restated by streamk_model.ring) plus the 1 KB reserved per CTA must fit twice
into the SM's 228 KB.
"""
import os
import re
import shutil
import subprocess

import pytest

from streamk_model import MAX_STAGES, RESERVED_PER_CTA, SMEM_PER_SM, ring, ring_smem  # noqa: F401 (re-exported)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so")

# Fmt with DECODE_2CTA whose decode tiles this file checks: the kernel's name -> streamk_model's format
FORMATS = {"Int4Fmt": "int4", "SsFmt<0>": "int8"}


def cfg(fmt, n_mma):
    """(stages, SMEM_BYTES) as ts_gemm.cuh Cfg<Fmt, N_MMA> computes them."""
    _, ctas, stages, _ = ring(FORMATS[fmt], n_mma)
    assert ctas == 2
    return stages, ring_smem(FORMATS[fmt], n_mma)


def resource_usage():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libao_b200.so not built")
    out = subprocess.run([exe, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    names = subprocess.run(["c++filt"], input=out, stdout=subprocess.PIPE, text=True).stdout if shutil.which("c++filt") else out
    usage = {}
    fn = None
    for line in names.splitlines():
        m = re.search(r"Function (.*ts_gemm_kernel<[^>]*?(\w+(?:<\d>)?), (\d+)>)", line)
        if m:
            fn = (m.group(2), int(m.group(3)))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            usage[fn] = (int(m.group(1)), int(m.group(2)))
            fn = None
    return usage


def test_stage_counts():
    want = {("Int4Fmt", 16): 7, ("Int4Fmt", 32): 6, ("SsFmt<0>", 16): 6, ("SsFmt<0>", 32): 5}
    for key, stages in want.items():
        assert cfg(*key)[0] == stages, key


@pytest.mark.parametrize("fmt", sorted(FORMATS))
@pytest.mark.parametrize("n_mma", [16, 32])
def test_two_decode_ctas_fit_per_sm(fmt, n_mma):
    stages, smem = cfg(fmt, n_mma)
    assert stages >= 2
    assert 2 * (smem + RESERVED_PER_CTA) <= SMEM_PER_SM
    usage = resource_usage()
    assert (fmt, n_mma) in usage, f"ts_gemm_kernel<{fmt}, {n_mma}> not in {LIB}"
    reg, stack = usage[(fmt, n_mma)]
    assert reg <= 80, f"ts_gemm_kernel<{fmt}, {n_mma}>: {reg} registers do not fit two 384-thread CTAs per SM"
    assert stack == 0, f"ts_gemm_kernel<{fmt}, {n_mma}>: {stack} bytes of stack (register spills)"
