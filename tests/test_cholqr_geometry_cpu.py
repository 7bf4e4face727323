"""The geometry mirror of the CholeskyQR2 compression (tests/cholqr_geometry.py): its invariants over every m up to 60 000
on cards of several sizes, and the coverage of tests/test_gpu_cholqr_geometry.py's route list."""
import pytest

from tests import cholqr_geometry as geo
from tests import test_gpu_cholqr_geometry as gpu_cases

SM_COUNTS = (132, 114, 66, 16, 1)  # H100 SXM, H100 PCIe, and smaller slices
# one n per (instance, BW) class: nt = 8 | 33 ; 64 | 65 ; 81 | 97 ; 121 | 129
CLASS_N = (7, 32, 63, 64, 80, 96, 120, 128)


def test_class_n_cover_every_class():
    classes = {(geo.instance_of(n + 1), (n + 1 + 31) // 32) for n in CLASS_N}
    assert classes == {((5, 0), 1), ((5, 0), 2), ((10, 0), 2), ((10, 0), 3), ((10, 5), 3), ((10, 5), 4), ((10, 10), 4), ((10, 10), 5)}


@pytest.mark.parametrize("sm", SM_COUNTS)
@pytest.mark.parametrize("n", CLASS_N)
def test_narrow_geometry_invariants(n, sm):
    seen = set()
    for m in range(1, 60001):
        g = geo.narrow_geometry(m, n, sm)
        assert g.smem_bytes <= geo.CQ_SG_SMEM
        assert g.cb % 4 == 0 and 0 < g.cb <= geo.ROUND_ROWS
        assert g.slab_rows % 4 == 0 and g.nslab >= 1 and 1 <= g.last_rows <= g.slab_rows
        assert (g.nslab - 1) * g.slab_rows + g.last_rows == m
        for rows, rounds in ((min(g.slab_rows, m), g.first), (g.last_rows, g.last)):
            if (rows, g.cb, g.ntail) in seen:
                continue
            seen.add((rows, g.cb, g.ntail))
            for nbuf, ntail in set(rounds):  # a long slab repeats its full-buffer round
                assert nbuf % 4 == 0 and 0 < nbuf <= g.cb
                assert ntail % 4 == 0 and nbuf + ntail <= geo.ROUND_ROWS  # 16 warps x 8 rows
                if ntail:
                    assert nbuf % 8 == 0  # row groups do not straddle buffer and scratch
                    assert ntail <= g.ntail  # within the scratch reserved per slab
            assert all(ntail == 0 for _, ntail in rounds[:-1])  # only the last round can split
            covered = sum(a + b for a, b in rounds)
            assert covered - sum(rounds[-1]) < rows  # only the last round is padded
            assert 0 <= covered - rows < 4  # the rounds tile the slab, padded to a whole k-step


@pytest.mark.parametrize("sm", SM_COUNTS)
@pytest.mark.parametrize("n", [160, 255, 256, 257, 383, 384, 385, 511, 512])
def test_wide_geometry_invariants(n, sm):
    for m in range(1, 20001):
        g = geo.wide_geometry(m, n, sm)
        assert g.slab_rows % 4 == 0 and 1 <= g.last_rows <= g.slab_rows
        assert (g.nslab - 1) * g.slab_rows + g.last_rows == m
        assert g.nslab * g.nblk <= max(sm, g.nblk)


def _cell_exists(inst, route, sm):
    return any(gpu_cases.route_m(n, route, sm) is not None for n in CLASS_N + (119, 159) if geo.instance_of(n + 1) == inst)


@pytest.mark.parametrize("sm", [132, 114])
def test_gpu_route_list_covers_every_cell(sm):
    """Every (instance x route) cell that some shape reaches has a case in the GPU test's list, and every listed case
    reaches its route."""
    listed = {(geo.instance_of(n + 1), r) for n, r in gpu_cases.NARROW_CASES}
    for inst in geo.INSTANCES:
        for route in geo.ROUTES:
            if _cell_exists(inst, route, sm):
                assert (inst, route) in listed, (inst, route)
    for n, route in gpu_cases.NARROW_CASES:
        m = gpu_cases.route_m(n, route, sm)
        assert m is not None, (n, route)
        assert route in geo.routes(geo.narrow_geometry(m, n, sm))
