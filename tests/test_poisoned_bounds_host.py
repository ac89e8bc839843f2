"""The poisoned arenas of tests/poison_arena.py on the CPU: carve() puts the view where it says and poisons every other
byte, intact() finds one flipped poison byte wherever it is, and two stand-ins for a faulty kernel are caught under the
poison meant for them (and only under it, which is why every GPU case runs under both)."""
import pytest
import torch

import poison_arena as pa

DEV = "cpu"


def _bytes_at(arena, offset, n):
    return arena.buf[offset:offset + n].tolist()


@pytest.mark.parametrize("poison", pa.POISONS)
@pytest.mark.parametrize("dtype,kind", [(torch.bfloat16, "bf16"), (torch.float32, "f32"), (torch.uint8, "e8m0"),
                                        (torch.int8, "i8"), (torch.int32, "int4")])
def test_carve_places_the_view_inside_poison(poison, dtype, kind):
    rows, cols, pitch = 5, 24, 40
    a = pa.carve((rows, cols), dtype, pitch=pitch, before=100, after=48, poison=poison, kind=kind, device=DEV)
    elem = a.view.element_size()
    assert a.view.shape == (rows, cols) and a.view.stride() == (pitch, 1)
    assert a.view.data_ptr() % 16 == 0
    assert a.view.data_ptr() - a.buf.data_ptr() == a.start == 112   # 100 rounded up to 16
    assert a.end == a.start + rows * pitch * elem and a.buf.numel() >= a.end + 48
    size, value = pa.pattern(kind, poison)
    want = list(value.to_bytes(size, "little"))
    # every element outside the view, and every element of the fresh view, holds the pattern
    assert a.buf.numel() % size == 0
    for off in range(0, a.buf.numel(), size):
        assert _bytes_at(a, off, size) == want, off
    assert int(a.guard.sum()) == a.buf.numel() - rows * cols * elem
    # writing the view leaves intact() satisfied; the gap columns are guarded, the row bytes are not
    a.view.copy_(torch.zeros(rows, cols, dtype=dtype))
    assert pa.intact(a) is None
    assert not bool(a.guard[a.start:a.start + cols * elem].any())
    assert bool(a.guard[a.start + cols * elem:a.start + pitch * elem].all())


def test_dense_and_multidimensional_views():
    a = pa.carve((3, 4, 8), torch.int32, poison="big", kind="int4", device=DEV)
    assert a.view.shape == (3, 4, 8) and a.view.is_contiguous()
    assert bool((a.view == -1).all())   # 0xFFFFFFFF
    b = pa.carve_like(torch.arange(6, dtype=torch.float32).reshape(2, 3), pitch=8)
    assert b.view.tolist() == [[0, 1, 2], [3, 4, 5]] and b.view.stride() == (8, 1)
    assert bool(torch.isnan(b.buf.view(torch.float32)[:4]).all())


@pytest.mark.parametrize("where", ["before", "after", "gap"])
def test_intact_finds_one_flipped_poison_byte(where):
    rows, cols, pitch = 4, 16, 24
    a = pa.carve((rows, cols), torch.bfloat16, pitch=pitch, poison="big", device=DEV)
    a.view.fill_(1.0)
    assert pa.intact(a) is None
    if where == "before":
        off, expect = a.start - 3, "before the view"
    elif where == "after":
        off, expect = a.end + 7, "past the view's end"
    else:   # row 2, element 20 of its pitch: a gap column
        off, expect = a.start + (2 * pitch + 20) * 2 + 1, "row 2"
    a.buf[off] ^= 0x01
    msg = pa.intact(a)
    assert msg is not None and expect in msg, msg
    if where == "gap":
        assert "byte 41 of row 2" in msg, msg


def test_fill_poisons_rows_of_the_view():
    a = pa.carve((6, 8), torch.bfloat16, poison="nan", device=DEV)
    a.view.fill_(2.0)
    a.fill(slice(4, None))
    assert bool(torch.isnan(a.view[4:].float()).all()) and bool((a.view[:4] == 2.0).all())
    assert pa.intact(a) is None


# ---------------------------------------------------------------------------------------------------- faulty kernels
def _strided_rows(poison, M=6, K=200, pitch=264):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(M, K, generator=g) * 3).to(torch.bfloat16)
    return pa.carve_like(x, pitch=pitch, poison=poison), x


def _fmax_rows(t):
    """A row amax as a kernel computes it with fmaxf: a NaN operand is dropped."""
    out = torch.zeros(t.shape[0], dtype=torch.float32)
    for j in range(t.shape[1]):
        out = torch.fmax(out, t[:, j].float().abs())
    return out


def _amax_over_pitch(arena):
    """Stand-in for a row amax whose loop runs over ldx / 8 vectors instead of K / 8."""
    pitch = arena.pitch_bytes // 2
    rows = arena.buf[arena.start:arena.end].view(torch.bfloat16).view(-1, pitch)
    return _fmax_rows(rows)


@pytest.mark.parametrize("poison", pa.POISONS)
def test_an_amax_over_the_pitch_is_caught_under_big(poison):
    a, x = _strided_rows(poison)
    right, wrong = _fmax_rows(x), _amax_over_pitch(a)
    assert torch.equal(_fmax_rows(a.view), right)
    caught = not torch.equal(wrong, right)
    # a huge finite gap moves the max; fmaxf drops a NaN gap, so that one goes unseen
    assert caught == (poison == "big")


def _k_tail_product(arena, w, chunk=128):
    """Stand-in for a K-tail chunk that reads x's row-pitch gap instead of zero fill: x rows over round_up(K, chunk)
    columns of the buffer, times w zero-filled past K."""
    K = arena.row_bytes // 2
    kp = -(-K // chunk) * chunk
    pitch = arena.pitch_bytes // 2
    assert pitch >= kp
    rows = arena.buf[arena.start:arena.end].view(torch.bfloat16).view(-1, pitch)[:, :kp].float()
    wz = torch.nn.functional.pad(w.float(), (0, kp - K))
    return rows @ wz.t()


@pytest.mark.parametrize("poison", pa.POISONS)
def test_a_k_tail_that_reads_the_gap_is_caught_under_nan(poison):
    a, x = _strided_rows(poison)
    w = torch.randn(8, x.shape[1], generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    right, wrong = x.float() @ w.float().t(), _k_tail_product(a, w)
    assert torch.equal(a.view.float() @ w.float().t(), right)
    caught = not torch.equal(wrong, right)
    # NaN x 0 is NaN; a huge finite value x 0 is 0
    assert caught == (poison == "nan")
