"""The HQQ restatement (tests/hqq_model.py) on the CPU: against the reference's own solves (golden fixtures
int4_hqq.npz and int4_hqq_shrink.npz) and the C oracle within the solver bars, and proof that the shrink fixture can
tell a dropped or sign-flipped shrinkage step apart, which the LLM-scale fixtures cannot.

The CPU restatement uses the CPU's powf, so it is a solve that differs from the reference's in the last bits, like the
oracle: it is held to the same bars (hqq_model.BARS).  Measured on int4_hqq_shrink.npz, restatement against the
reference: scales equal, codes 0.55 % different at most, zero points 0.8 % different in their bits and 0.6 % more than
0.01 step apart at most, reconstruction error within 2e-4; oracle against the reference: zero points 2.3 % different in
their bits at most, everything else as the restatement.
"""
import ctypes
import os

import numpy as np
import pytest

import hqq_model as hm
from oracle import oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = {"int4_hqq.npz": ("g32", "g128", "g64_outlier"),
            "int4_hqq_shrink.npz": ("s002_g256", "s1_g32", "s1_g256", "s2_g128")}
SHRINK_CASES = ("s1_g32", "s1_g256", "s2_g128")
CASES = [(f, c) for f, cs in FIXTURES.items() for c in cs]


def _load(golden_dir, fixture, case):
    d = np.load(os.path.join(golden_dir, fixture))
    return d[f"{case}__w"], int(d[f"{case}__g"]), d[f"{case}__q"], d[f"{case}__s"], d[f"{case}__z"]


def _solve(w_bits, g, **kw):
    r = hm.solve(o.bf16_tensor(w_bits), g, **kw)
    return r, (r.q.numpy(), o.bf16_bits(r.scale), o.bf16_bits(r.zero))


@pytest.mark.parametrize("fixture,case", CASES)
def test_restatement_matches_reference_within_solver_bars(golden_dir, fixture, case):
    w, g, qr, sr, zr = _load(golden_dir, fixture, case)
    r, out = _solve(w, g)
    rep = hm.bar_report(w, g, *out, qr, sr, zr)
    assert hm.within_bars(rep), rep
    assert 1 <= r.iters <= hm.ITERS and (r.stop == 1 or r.iters == hm.ITERS)


@pytest.mark.parametrize("fixture,case", CASES)
def test_restatement_matches_oracle_within_solver_bars(golden_dir, fixture, case):
    w, g, *_ = _load(golden_dir, fixture, case)
    qo, so, zo, iters = o.int4_hqq(w, g)
    r, out = _solve(w, g)
    rep = hm.bar_report(w, g, *out, qo, so, zo)
    assert hm.within_bars(rep), rep
    assert r.iters == iters


@pytest.mark.parametrize("case", SHRINK_CASES)
@pytest.mark.parametrize("mutation", ["no_shrink", "flip_sign"])
def test_shrink_fixture_tells_a_broken_shrinkage_step_apart(golden_dir, case, mutation):
    """A solve without the shrinkage step, or with its sign flipped, passes the bars on the LLM-scale fixtures (the
    step never switches on there) but fails them on every shrink-active case."""
    w, g, qr, sr, zr = _load(golden_dir, "int4_hqq_shrink.npz", case)
    r, out = _solve(w, g, **{mutation: True})
    rep = hm.bar_report(w, g, *out, qr, sr, zr)
    assert not hm.within_bars(rep), (mutation, rep)


@pytest.mark.parametrize("fixture,case", CASES)
def test_tier1_classifier(golden_dir, fixture, case):
    """Tier 1 (the relu is zero whatever the last bits of powf) accepts every LLM-scale case and rejects every
    shrink-active one.  On the LLM-scale fixtures no element is ever shrunk, which is why they cannot tell a broken
    shrinkage step apart and the shrink fixture exists."""
    w, g, *_ = _load(golden_dir, fixture, case)
    r, _ = _solve(w, g)
    if case in SHRINK_CASES:
        assert not r.tier1 and min(r.active) > 0, (r.margin, r.active)
    else:
        assert r.tier1 and sum(r.active) == 0, (r.margin, r.active)


@pytest.mark.parametrize("g", [32, 256])
def test_tier1_holds_for_llm_scale_weights(g):
    for regime in ("s002", "s002_outlier"):
        r = hm.solve(hm.weight(regime, 128, 2048, g), g)
        assert r.tier1 and sum(r.active) == 0, (regime, r.margin)
    r = hm.solve(hm.weight("s1", 128, 2048, g), g)
    assert not r.tier1 and min(r.active) > 0


def test_workspace_layout_fits_the_declared_workspace():
    """hqq_model.workspace_layout is where the tests read the solver's state: scale[G], zero[G], partial[nblocks]
    doubles at align16(8 G), then Ctrl {double best; int stop; int iters}."""
    lib = ctypes.CDLL(os.path.join(ROOT, "ao_b200", "lib", "libao_b200.so"))
    lib.ao_int4_hqq_workspace_bytes.restype = ctypes.c_size_t
    for N, K, g in [(3, 96, 32), (64, 1024, 32), (1032, 4096, 256), (6144, 4096, 32), (4096, 14336, 128)]:
        G, nb, off_p, off_c = hm.workspace_layout(N, K, g)
        assert off_p >= 8 * G and off_p % 16 == 0 and off_c == off_p + 8 * nb
        assert off_c + 16 <= lib.ao_int4_hqq_workspace_bytes(N, K, g)
