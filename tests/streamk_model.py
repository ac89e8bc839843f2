"""A CPU restatement of the stream-K work split of the quantized GEMM kernel, for tests.

It mirrors `unit_begin`, `cta_of_unit` and `Walk` of ao_b200/csrc/streamk.cuh, the grid choice and the partial
group width `GB` of ao_b200/csrc/ts_gemm.cuh, and the token-tile width and K-chunk count each launcher picks.  Keep
the two in step: a change to the walk there needs the same change here, or test_streamk_plan.py and the messages of
test_exact_gemm_gpu.py describe a split the kernel does not run.
"""
from dataclasses import dataclass, field

ROWS = 128        # weight rows of a tile
KCHUNK = 128      # k of a unit
FULL, CONTRIB, OWNER = 0, 1, 2
KIND_NAMES = {FULL: "FULL", CONTRIB: "CONTRIB", OWNER: "OWNER"}

# token-tile widths each format's launcher can pick (fp8 keeps a second accumulator per chunk: 64 at most)
WIDTHS = {"int4": (16, 32, 64, 128), "int8": (16, 32, 64, 128), "fp8": (16, 32, 64), "mxfp8": (16, 32, 64, 128),
          "nvfp4": (16, 32, 64, 128)}


def n_mma(fmt, M):
    for w in WIDTHS[fmt]:
        if M <= w:
            return w
    return WIDTHS[fmt][-1]


def k_chunks(fmt, K):
    # int4 / nvfp4 need K % 128 == 0 (K / 128); the 8-bit kinds zero-fill a K tail (ceil)
    return -(-K // KCHUNK)


def group_width(width):
    """GB of the owner's gather (ts_gemm.cuh): partials of GB contributors are loaded before any is added."""
    nacc = width // 2
    return 4 if nacc <= 8 else (2 if nacc <= 16 else 1)


def unit_begin(b, U, G):
    return (U * b) // G


def cta_of_unit(u, U, G):
    return ((u + 1) * G + U - 1) // U - 1


def default_grid(units, sm=132, min_units=4):
    grid = sm
    if units // min_units < grid:
        grid = units // min_units if units // min_units > 0 else 1
    return grid


def forced_grid(n, units, sm=132):
    """launch_gemm under ao_b200_debug_set_streamk_ctas(n), n > 0."""
    return max(1, min(n, sm, units))


@dataclass
class Seg:
    tile: int
    kc0: int      # first chunk of the segment within its tile
    count: int
    kind: int


def walk(u0, nunits, KT):
    """Walk of streamk.cuh: the segments of the unit range [u0, u0 + nunits)."""
    kc0 = u0 % KT
    cnt0 = min(KT - kc0, nunits)
    nseg = 1 + (nunits - cnt0 + KT - 1) // KT
    segs = []
    for s in range(nseg):
        begin = 0 if s == 0 else cnt0 + (s - 1) * KT
        count = cnt0 if s == 0 else min(nunits - begin, KT)
        if count == KT:
            kind = FULL
        elif s == 0 and kc0 != 0:
            kind = CONTRIB
        else:
            kind = OWNER
        segs.append(Seg(u0 // KT + s, kc0 if s == 0 else 0, count, kind))
    return segs


@dataclass
class Plan:
    fmt: str
    M: int
    N: int
    K: int
    G: int
    width: int
    n_tiles: int
    m_blocks: int
    KT: int
    U: int
    ctas: list = field(default_factory=list)        # ctas[b] = list of Seg
    owners: dict = field(default_factory=dict)      # split tile -> (owner CTA, [contributor CTAs])

    @property
    def gb(self):
        return group_width(self.width)

    def contributor_counts(self):
        return [len(c) for _, c in self.owners.values()]

    def tile_of(self, m, n):
        return (m // self.width) * self.n_tiles + n // ROWS

    def describe(self, m, n):
        """The tile of output (m, n) and the CTAs and segment kinds that computed it."""
        t = self.tile_of(m, n)
        parts = []
        for b in range(cta_of_unit(t * self.KT, self.U, self.G), cta_of_unit(t * self.KT + self.KT - 1, self.U, self.G) + 1):
            for s in self.ctas[b]:
                if s.tile == t:
                    parts.append(f"CTA {b} {KIND_NAMES[s.kind]} chunks {s.kc0}..{s.kc0 + s.count - 1}")
        return (f"tile {t} (n-tile {t % self.n_tiles}, m-block {t // self.n_tiles}) of {self.fmt} M={self.M} N={self.N} "
                f"K={self.K} N_MMA={self.width} grid={self.G}: " + "; ".join(parts))


def plan(fmt, M, N, K, grid=None, sm=132):
    """The split the kernel runs for one launch.  grid: None = the default heuristic on `sm` SMs, else the forced
    CTA count (clamped like launch_gemm).  N is the number of output features the kernel tiles (int4: N_out)."""
    width = n_mma(fmt, M)
    KT = k_chunks(fmt, K)
    n_tiles, m_blocks = -(-N // ROWS), -(-M // width)
    U = n_tiles * m_blocks * KT
    G = default_grid(U, sm) if grid is None else forced_grid(grid, U, sm)
    p = Plan(fmt, M, N, K, G, width, n_tiles, m_blocks, KT, U)
    for b in range(G):
        u0, u1 = unit_begin(b, U, G), unit_begin(b + 1, U, G)
        p.ctas.append(walk(u0, u1 - u0, KT) if u1 > u0 else [])
    for b, segs in enumerate(p.ctas):
        if segs and segs[-1].kind == OWNER:
            t = segs[-1].tile
            b_last = cta_of_unit(t * KT + KT - 1, U, G)
            p.owners[t] = (b, list(range(b + 1, b_last + 1)))
    return p
