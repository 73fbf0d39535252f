"""CPU: the PME entry points of include/spk_b200.h are exported by the library and bound by _lib, with their launch
counts and the workspace formula of csrc/pme.cu."""
import ctypes

import pytest


def test_pme_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ("spk_pme_workspace_bytes", "spk_pme_spread", "spk_pme_energy", "spk_pme_bwd"):
        assert hasattr(h, name), name
        assert name in _lib.SIGNATURES
    assert _lib.SIGNATURES["spk_pme_workspace_bytes"] == [ctypes.c_int64] * 5 + [ctypes.c_int]
    assert len(_lib.SIGNATURES["spk_pme_spread"]) == 15
    assert len(_lib.SIGNATURES["spk_pme_energy"]) == 17
    assert len(_lib.SIGNATURES["spk_pme_bwd"]) == 23
    # spread: cell, setup, frac, bin, scan, fill, sort, spread; energy: influence, energy; reverse: gather, per system
    assert (_lib.LAUNCHES["spk_pme_spread"], _lib.LAUNCHES["spk_pme_energy"], _lib.LAUNCHES["spk_pme_bwd"]) == (8, 2, 2)


def _expected(N, B, n1, n2, n3):
    """doubles: system records 16 B, fractions 3 N, moduli n1 + n2 + n3, energies 8 B, 7-wide partials of the frequency
    pass and 9-wide partials of the atom pass; int32: keys and sorted atoms 2 N, counts, cursors and bin starts
    3 B bricks + 1, frequency starts B + 1 (rounded up to whole doubles)"""
    cd = lambda a, b: -(-a // b)
    F = n1 * n2 * (n3 // 2 + 1)
    nb = cd(n1, 8) * cd(n2, 8) * cd(n3, 8)
    dbl = 16 * B + 3 * N + n1 + n2 + n3 + 8 * B + 7 * (B + cd(B * F, 128) + 1) + 9 * (B + cd(N, 128) + 1)
    ints = 2 * N + 3 * B * nb + 1 + B + 1
    return 8 * (dbl + (ints + 1) // 2)


@pytest.mark.parametrize("N,B,mesh,order", [(1, 1, (8, 8, 8), 8), (300, 4, (45, 48, 50), 4), (8192, 1, (48, 48, 48), 6),
                                            (0, 2, (6, 7, 9), 6)])
def test_pme_workspace_formula(N, B, mesh, order):
    from schnetpack_b200 import _lib

    assert _lib.lib().spk_pme_workspace_bytes(N, B, *mesh, order) == _expected(N, B, *mesh)


def test_pme_workspace_refuses_bad_order_and_mesh():
    from schnetpack_b200 import _lib

    ws = _lib.lib().spk_pme_workspace_bytes
    assert ws(10, 1, 16, 16, 16, 5) == 0 and ws(10, 1, 16, 16, 16, 10) == 0
    assert ws(10, 1, 16, 7, 16, 8) == 0 and ws(10, 1, 16, 16, 16, 8) > 0
