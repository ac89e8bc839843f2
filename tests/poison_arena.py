"""Poisoned neighbourhoods for kernel operands: a view inside a larger buffer whose every other byte is poison.

carve() places a tensor view, 16-byte aligned as the ops require, inside a buffer that holds poison before it, after
it and, when the row pitch is wider than a row, in the gap columns between its rows.  intact() reports the first
poison byte that changed.  A kernel that reads past an operand then reads poison, and one that writes past an output
overwrites it.

Two poisons per element kind, and each case runs under both: "nan" feeds a NaN (or the other extreme, for kinds
without one) into any product an over-read reaches, "big" feeds a huge finite value into any max or sum.  A NaN is not
enough alone: fmaxf drops it, so an amax that runs into a NaN gap is unchanged, and a huge finite value times a
zero-filled weight is 0.

    kind   "nan"                "big"
    bf16   0x7FC0               0x7F7F (max finite)
    f32    0x7FC00000           3.0e38
    e4m3   0x7F                 0x7E (448)
    e8m0   0xFF                 0xFE (2^127)
    i8     0x80 (-128)          0x7F (127)
    fp4    0xFF (-6, -6)        0x77 (6, 6)              packed e2m1 pairs
    int4   0x00000000 (-8 x 8)  0xFFFFFFFF (+7 x 8)      tile-packed int4 words: every nibble at an extreme
    i32    0x80000000           0x7FFFFFFF
    u8     0xFF                 0xFE                     other bytes (NF4 codes, 2:4 metadata)
"""
import struct

import torch

POISONS = ("nan", "big")
ALIGN = 16

_F32_BIG = struct.unpack("<I", struct.pack("<f", 3.0e38))[0]
# kind: (element bytes, "nan" pattern, "big" pattern)
PATTERNS = {
    "bf16": (2, 0x7FC0, 0x7F7F),
    "f32": (4, 0x7FC00000, _F32_BIG),
    "e4m3": (1, 0x7F, 0x7E),
    "e8m0": (1, 0xFF, 0xFE),
    "i8": (1, 0x80, 0x7F),
    "fp4": (1, 0xFF, 0x77),
    "int4": (4, 0x00000000, 0xFFFFFFFF),
    "i32": (4, 0x80000000, 0x7FFFFFFF),
    "u8": (1, 0xFF, 0xFE),
}
_DEFAULT_KIND = {torch.bfloat16: "bf16", torch.float32: "f32", torch.float8_e4m3fn: "e4m3", torch.int8: "i8",
                 torch.int32: "i32", torch.uint8: "u8", torch.int16: "bf16"}
_INT_OF_SIZE = {1: torch.uint8, 2: torch.int16, 4: torch.int32}


def _signed(value, size):
    """The bit pattern `value` as the signed integer torch fills an int dtype of `size` bytes with."""
    if size == 1:
        return value
    top = 1 << (8 * size)
    return value - top if value >= top // 2 else value


def pattern(kind, poison):
    size, nan, big = PATTERNS[kind]
    return size, (nan if poison == "nan" else big)


def _round_up(v, a):
    return -(-v // a) * a


class Arena:
    """view: the operand, `shape` elements with row pitch `pitch` (elements) when given; buf: the whole uint8 buffer.
    [start, end) is the byte span from the view's first row to the end of its last row's pitch."""

    def __init__(self, buf, view, start, end, guard, snapshot, kind, poison, row_bytes, pitch_bytes):
        self.buf, self.view, self.start, self.end = buf, view, start, end
        self.guard, self.snapshot = guard, snapshot
        self.kind, self.poison = kind, poison
        self.row_bytes, self.pitch_bytes = row_bytes, pitch_bytes

    def fill(self, index=slice(None)):
        """Writes the poison into view[index] (rows the operation must not read, or an output before a launch)."""
        size, value = pattern(self.kind, self.poison)
        v = self.view
        if v.element_size() != size:
            raise ValueError(f"{self.kind} poison on {v.dtype} elements")
        v.view(_INT_OF_SIZE[size])[index] = _signed(value, size)
        return self

    def where(self, offset):
        """Describes byte `offset` of buf: its side of the view and its offset from the view's start."""
        if offset < self.start:
            return f"byte {offset - self.start} (before the view)"
        if offset >= self.end:
            return f"byte +{offset - self.end} past the view's end"
        rel = offset - self.start
        return f"byte {rel % self.pitch_bytes} of row {rel // self.pitch_bytes} (a gap column: row bytes {self.row_bytes})"


def carve(shape, dtype, pitch=None, before=256, after=256, poison="nan", kind=None, device="cuda"):
    """A view of `shape` elements of `dtype` inside a poisoned buffer.  pitch: row pitch in elements of a 2-D view
    (None: dense rows); before / after: poison bytes on either side (rounded up to 16).  Every byte outside the view
    holds the poison of `kind` (default: from dtype), the view included until written.  Returns an Arena."""
    kind = kind or _DEFAULT_KIND[dtype]
    size, value = pattern(kind, poison)
    elem = torch.empty((), dtype=dtype).element_size()
    assert elem == size, f"{kind} poison is {size}-byte, {dtype} elements are {elem}"
    shape = tuple(int(s) for s in shape)
    rows = shape[0] if shape else 1
    cols = 1
    for s in shape[1:]:
        cols *= s
    if pitch is None:
        pitch = cols
    else:
        assert len(shape) == 2 and pitch >= cols, "a pitch is a 2-D view's row stride, at least its row length"
    row_bytes, pitch_bytes = cols * elem, pitch * elem
    span = rows * pitch_bytes
    before, after = _round_up(before, ALIGN), _round_up(after, ALIGN)
    buf = torch.empty(_round_up(before + span + after, ALIGN), dtype=torch.uint8, device=device)
    assert buf.data_ptr() % ALIGN == 0, "allocations start on 16 bytes"
    start = before
    # the pattern on element boundaries counted from offset 0, so from the view's start as well
    buf.view(_INT_OF_SIZE[size]).fill_(_signed(value, size))
    flat = buf[start:start + span].view(dtype)
    if pitch == cols:
        view = flat.view(shape) if shape else flat.view(())
    else:
        view = flat.view(rows, pitch)[:, :cols]
    assert view.data_ptr() % ALIGN == 0
    guard = torch.ones(buf.numel(), dtype=torch.bool, device=device)
    body = guard[start:start + span].view(rows, pitch_bytes)
    body[:, :row_bytes] = False
    return Arena(buf, view, start, start + span, guard, buf.clone(), kind, poison, row_bytes, pitch_bytes)


def carve_like(t, pitch=None, poison="nan", kind=None, before=256, after=256):
    """carve() of t's shape and dtype with t's values copied into the view."""
    a = carve(t.shape, t.dtype, pitch=pitch, poison=poison, kind=kind, before=before, after=after, device=t.device)
    a.view.copy_(t)
    return a


def intact(arena):
    """None when every poison byte of the arena is unchanged, else a description of the first changed one."""
    changed = (arena.buf != arena.snapshot) & arena.guard
    if not bool(changed.any()):
        return None
    idx = changed.nonzero().flatten()
    first = int(idx[0])
    return (f"{int(idx.numel())} poison bytes changed, first {arena.where(first)}: "
            f"{int(arena.snapshot[first]):#04x} -> {int(arena.buf[first]):#04x}")
