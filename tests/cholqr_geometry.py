"""Pure-Python mirror of the host-side geometry of the CholeskyQR2 compression (csrc/k_cholqr.cu), so that tests can
choose shapes that reach a given slab / round route of k_cq_solve_gram on whatever GPU they run on.

Mirrored, line for line:
  launch_compress_cholqr2  slab sizing of the narrow path (nt <= CQ_MAXN)      k_cholqr.cu:1280-1288
  cq_launch_solve_gram     template instance <NH1, NH2> from NB = ceil(nt / 8)  k_cholqr.cu:843-851
  cq_sg_pitch              buffer pitch                                         k_cholqr.cu:706-709
  cq_sg_shape              buffer rows cb and the reserved scratch rows ntail   k_cholqr.cu:816-825
  k_cq_solve_gram          the round loop of one slab (split_at, nbuf_at, ntail) k_cholqr.cu:757-765
  cq_compress_wide         slab sizing of the blocked path (nt <= 513)          k_cholqr.cu:1228-1239
A change to any of them has to be repeated here; tests/test_cholqr_geometry_cpu.py checks the mirror's invariants.
"""
from __future__ import annotations

from functools import lru_cache
from typing import NamedTuple

CQ_MAXN = 160
CQ_MAXB = 20
CQ_KB = 32
CQ_GRAM_T = 512
ROUND_ROWS = 8 * (CQ_GRAM_T // 32)  # one 8-row group per warp: the most rows one round solves
CQ_PK_INV = (CQ_MAXB * (CQ_MAXB + 1) // 2) * 64
CQ_PK_DOUBLES = CQ_PK_INV + CQ_MAXB * 8
CQ_SG_SMEM = 226 * 1024
CQ_WB = 128
CQ_WMAX = 520

INSTANCES = ((5, 0), (10, 0), (10, 5), (10, 10))

# routes of the narrow path (see routes()); the split routes exist only where cb < ROUND_ROWS
ROUTES = ("single", "multi", "split", "multi_split", "tail_min", "tail_max", "last_1", "last_2", "last_3", "one_slab", "m_le_n")
SPLIT_ROUTES = ("split", "multi_split", "tail_min", "tail_max")


def instance_of(nt: int) -> tuple[int, int]:
    NB = (nt + 7) // 8
    return (5, 0) if NB <= 5 else (10, 0) if NB <= 10 else (10, 5) if NB <= 15 else (10, 10)


def sg_pitch(BW: int, NBP: int) -> int:
    w = max(8 * NBP, 32 * BW)
    return ((w + 15) & ~15) + 4


@lru_cache(maxsize=None)
def sg_shape(nt: int, BW: int, slab_rows: int) -> tuple[int, int, int]:
    """(pitch, cb, ntail) of cq_sg_shape."""
    NBP = sum(instance_of(nt))
    pitch = sg_pitch(BW, NBP)
    rnd = min(slab_rows, ROUND_ROWS)
    fit = ((CQ_SG_SMEM - 8 * CQ_PK_DOUBLES) // (8 * pitch)) & ~3
    cb = min(fit, rnd)
    ntail = rnd - (cb & ~7) if slab_rows > cb else 0
    return pitch, cb, ntail


@lru_cache(maxsize=None)
def slab_rounds(rows: int, cb: int) -> tuple[tuple[int, int], ...]:
    """(nbuf, ntail) of every round k_cq_solve_gram runs over a slab of `rows` rows (r1 - r0) with a buffer of cb rows."""
    # while more than ROUND_ROWS rows are left, every round fills the buffer (nbuf = cb, no split): taken in one step
    full = max(0, -(-(rows - ROUND_ROWS) // cb))
    out = [(cb, 0)] * full
    rc = full * cb
    while rc < rows:
        left = rows - rc
        split = cb < left <= ROUND_ROWS  # split_at
        nbuf = (cb & ~7) if split else min(cb, (left + 3) & ~3)  # nbuf_at
        ntail = ((left - nbuf + 3) & ~3) if split else 0
        out.append((nbuf, ntail))
        rc += nbuf + ntail
    return tuple(out)


class NarrowGeometry(NamedTuple):
    m: int
    n: int
    sm_count: int
    instance: tuple[int, int]
    BW: int
    pitch: int
    cb: int
    ntail: int       # scratch rows reserved per slab
    slab_rows: int
    nslab: int
    last_rows: int   # rows of the last slab
    first: tuple     # (nbuf, ntail) rounds of the first slab (min(slab_rows, m) rows)
    last: tuple      # ... and of the last slab

    @property
    def smem_bytes(self) -> int:
        return 8 * (CQ_PK_DOUBLES + self.cb * self.pitch)


def narrow_geometry(m: int, n: int, sm_count: int) -> NarrowGeometry:
    nt = n + 1
    assert 1 <= m and nt <= CQ_MAXN
    BW = (nt + 31) // 32
    nslab = min(sm_count, (m + CQ_KB - 1) // CQ_KB)
    slab_rows = (((m + nslab - 1) // nslab) + 3) & ~3
    nslab = (m + slab_rows - 1) // slab_rows
    pitch, cb, ntail = sg_shape(nt, BW, slab_rows)
    last_rows = m - (nslab - 1) * slab_rows
    return NarrowGeometry(m, n, sm_count, instance_of(nt), BW, pitch, cb, ntail, slab_rows, nslab, last_rows,
                          slab_rounds(min(slab_rows, m), cb), slab_rounds(last_rows, cb))


@lru_cache(maxsize=None)
def _slab_routes(rows: int, cb: int) -> frozenset:
    rounds = slab_rounds(rows, cb)
    split = rounds[-1][1] > 0
    if len(rounds) == 1:
        r = {"split" if split else "single"}
    elif split:
        r = {"multi_split"}
    else:
        r = {"multi"} if rounds[-1][0] < cb else set()  # several rounds, all full: no partial last round
    if split:
        tail = rows - sum(a + b for a, b in rounds[:-1]) - rounds[-1][0]  # rows of the split round past the buffer
        if tail == cb + 1 - (cb & ~7):
            r.add("tail_min")
        if tail == ROUND_ROWS - (cb & ~7):
            r.add("tail_max")
    return frozenset(r)


def routes(g: NarrowGeometry) -> set[str]:
    """The routes of ROUTES a shape takes:
    single / split / multi / multi_split   a slab (first or last) of one plain round / one split round / several rounds
                                           ending in a partial (zero-padded) round / several rounds ending in a split
    tail_min / tail_max                    a split round with the fewest rows past the buffer (cb + 1 - (cb & ~7): three
                                           zero rows pad the scratch) / the longest scratch tail (a full ROUND_ROWS round)
    last_1..3                              a 1..3-row last slab behind full ones
    one_slab, m_le_n                       one slab; no more rows than columns"""
    r = set(_slab_routes(min(g.slab_rows, g.m), g.cb) | _slab_routes(g.last_rows, g.cb))
    if g.nslab > 1 and g.last_rows <= 3:
        r.add(f"last_{g.last_rows}")
    if g.nslab == 1:
        r.add("one_slab")
    if g.m <= g.n:
        r.add("m_le_n")
    return r


@lru_cache(maxsize=None)
def find_m(n: int, route: str, sm_count: int, m_min: int = 1) -> int | None:
    """Smallest m >= m_min whose (m, n) system takes `route` at sm_count SMs, or None. The search stops at slabs of 512
    rows: every round sequence (full rounds, then a partial or a split round) has occurred by then."""
    for m in range(m_min, max(m_min, 512 * sm_count) + 1):
        g = narrow_geometry(m, n, sm_count)
        if route in routes(g):
            return m
        if route == "m_le_n" and m > n:
            return None
        if route == "one_slab" and g.nslab > 1:
            return None
    return None


# ---------------------------------------------------------------------------------------------------------------- wide path
class WideGeometry(NamedTuple):
    m: int
    n: int
    nblk_side: int
    nblk: int
    nslab: int
    slab_rows: int
    last_rows: int
    chol_blocks: int  # CQ_WB-column blocks of the blocked Cholesky (the last one may be narrow)


def wide_geometry(m: int, n: int, sm_count: int) -> WideGeometry:
    nt = n + 1
    assert CQ_MAXN < nt <= CQ_WMAX - 7
    nT = (nt + 31) // 32
    nblk_side = (nT + 3) // 4
    nblk = nblk_side * (nblk_side + 1) // 2
    nslab = min(max(1, sm_count // nblk), (m + CQ_KB - 1) // CQ_KB)
    slab_rows = (((m + nslab - 1) // nslab) + 3) & ~3
    nslab = (m + slab_rows - 1) // slab_rows
    return WideGeometry(m, n, nblk_side, nblk, nslab, slab_rows, m - (nslab - 1) * slab_rows, (nt + CQ_WB - 1) // CQ_WB)


def find_m_wide(n: int, sm_count: int, m_min: int, pred) -> int | None:
    for m in range(m_min, m_min + 200_000):
        if pred(wide_geometry(m, n, sm_count)):
            return m
    return None
