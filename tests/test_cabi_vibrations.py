"""CPU: the vibrational-analysis entry points of include/spk_b200.h are exported by the library and bound by _lib (the
layout of spk_vib_t is checked with every other struct in test_cabi_library.py)."""
import ctypes

ENTRY_POINTS = ["spk_vib_displace", "spk_vib_assemble", "spk_vib_finish"]


def test_vibration_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ENTRY_POINTS:
        assert hasattr(h, name), name
        assert _lib.SIGNATURES[name] == [ctypes.POINTER(_lib.VibParams), _lib.P]
