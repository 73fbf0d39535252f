"""CPU: the FIRE entry points of include/spk_b200.h are exported by the library and bound by _lib (the layout of
spk_fire_t is checked with every other struct in test_cabi_library.py)."""
import ctypes


def test_fire_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ("spk_fire_workspace_bytes", "spk_fire_forces", "spk_fire_step"):
        assert hasattr(h, name), name
    assert _lib.SIGNATURES["spk_fire_forces"] == [ctypes.POINTER(_lib.FIREState), _lib.P, _lib.P, _lib.P]
    assert _lib.SIGNATURES["spk_fire_step"] == [ctypes.POINTER(_lib.FIREState), _lib.P]
    assert _lib.LAUNCHES["spk_fire_forces"] == 3 and _lib.LAUNCHES["spk_fire_step"] == 2
    assert _lib.FIREState.mask.size == 9 * ctypes.sizeof(ctypes.c_double)
    ws = _lib.lib().spk_fire_workspace_bytes
    assert ws(0, 1) == 3 * 8 and ws(257, 2) == 3 * 8 * (2 + 2)      # 3 sums per system and per CTA of 256 atoms
