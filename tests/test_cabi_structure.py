"""CPU: the structure entry points of include/spk_b200.h are exported by the library and bound by _lib, with their launch
counts and the workspace formulas of csrc/structure.cu."""
import ctypes

import pytest


def test_structure_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ("spk_rdf_workspace_bytes", "spk_rdf_accumulate", "spk_msd_workspace_bytes", "spk_msd_accumulate"):
        assert hasattr(h, name), name
        assert name in _lib.SIGNATURES
    assert _lib.SIGNATURES["spk_rdf_workspace_bytes"] == [ctypes.c_int64] * 4
    assert _lib.SIGNATURES["spk_msd_workspace_bytes"] == [ctypes.c_int64] * 4
    assert len(_lib.SIGNATURES["spk_rdf_accumulate"]) == 25
    assert len(_lib.SIGNATURES["spk_msd_accumulate"]) == 28
    # rdf: sampling flag, grid setup, bin, sort, cell bounds, traversal, fold; msd: flag, track, centre-of-mass partials
    # and finish, displacement partials and finish, advance
    assert (_lib.LAUNCHES["spk_rdf_accumulate"], _lib.LAUNCHES["spk_msd_accumulate"]) == (7, 7)


def _msd_expected(N, B, S, K):
    """doubles: flag 1, centre-of-mass partials 4 B + 4 n_cta, centres 3 B, lags K, displacement partials
    K (B + n_cta) W with W = S rounded up to a power of two <= 8"""
    n_cta = -(-N // 256)
    W = 1 if S <= 1 else 2 if S <= 2 else 4 if S <= 4 else 8
    return 8 * (1 + 7 * B + 4 * n_cta + K + K * (B + n_cta) * W)


@pytest.mark.parametrize("N,B,S,K", [(1, 1, 1, 1), (300, 4, 3, 40), (24000, 1, 5, 7), (257, 2, 8, 3)])
def test_msd_workspace_formula(N, B, S, K):
    from schnetpack_b200 import _lib

    assert _lib.lib().spk_msd_workspace_bytes(N, B, S, K) == _msd_expected(N, B, S, K)


def test_msd_workspace_refuses_bad_species():
    from schnetpack_b200 import _lib

    ws = _lib.lib().spk_msd_workspace_bytes
    assert ws(10, 1, 0, 4) == 0 and ws(10, 1, 9, 4) == 0 and ws(10, 1, 3, 0) == 0 and ws(10, 1, 8, 4) > 0


@pytest.mark.parametrize("N,B,S,n_bins", [(1, 1, 1, 1), (3000, 1, 7, 400), (500, 4, 4, 100)])
def test_rdf_workspace_holds_the_grid_and_the_frame_counts(N, B, S, n_bins):
    """the neighbour-list grid (without its pair-count scan) plus one int32 count per (system, slot, bin)"""
    from schnetpack_b200 import _lib

    h = _lib.lib()
    ws = h.spk_rdf_workspace_bytes(N, B, S, n_bins)
    assert ws >= 4 * B * S * n_bins + 4 * 4 * N + 12 * N
    assert h.spk_rdf_workspace_bytes(N, B, S, n_bins + 64) - ws >= 4 * B * S * 64 - 255
    assert h.spk_rdf_workspace_bytes(-1, B, S, n_bins) == 0
