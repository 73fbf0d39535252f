"""CPU: the NEB entry points of include/spk_b200.h are exported by the library and bound by _lib (the layout of spk_neb_t
is checked with every other struct in test_cabi_library.py)."""
import ctypes


def test_neb_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ("spk_neb_workspace_bytes", "spk_neb_forces"):
        assert hasattr(h, name), name
    assert _lib.SIGNATURES["spk_neb_forces"] == [ctypes.POINTER(_lib.NEBState), _lib.P, _lib.P, _lib.P]
    assert _lib.SIGNATURES["spk_neb_workspace_bytes"] == [ctypes.c_int64, ctypes.c_int64]
    assert _lib.LAUNCHES["spk_neb_forces"] == 3
    ws = _lib.lib().spk_neb_workspace_bytes
    # 5 sums per interior image and per CTA of 256 atoms
    assert ws(1, 1) == 5 * 8 * (1 + 1) and ws(257, 3) == 5 * 8 * (3 + 2) and ws(20_000 * 7, 7) == 5 * 8 * (7 + 547)
