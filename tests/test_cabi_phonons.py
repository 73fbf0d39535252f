"""CPU: the phonon entry points of include/spk_b200.h are exported by the library and bound by _lib, and the
displaced-atom count of spk_vib_t is bound (the layouts of spk_ph_t and spk_vib_t are checked with every other struct in
test_cabi_library.py)."""
import ctypes
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ["spk_ph_force_constants", "spk_ph_images", "spk_ph_dynmat", "spk_ph_dos", "spk_ph_thermo",
                "spk_ph_thermo_workspace_bytes"]


def test_phonon_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ENTRY_POINTS:
        assert hasattr(h, name), name
        assert name in _lib.SIGNATURES, name
    assert _lib.SIGNATURES["spk_ph_force_constants"] == [ctypes.POINTER(_lib.PhononParams), _lib.P]
    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    assert f"#define SPK_PH_MAX_IMAGES {_lib.PH_MAX_IMAGES}" in text
    assert "n_displaced" in [f[0] for f in _lib.VibParams._fields_]


def test_thermo_workspace_formula():
    from schnetpack_b200 import _lib

    lib = _lib.lib()
    assert lib.spk_ph_thermo_workspace_bytes(1000, 7) == 8 * _lib.PH_THERMO_FIELDS * (7 + 4)
