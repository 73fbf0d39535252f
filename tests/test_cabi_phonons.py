"""CPU: the phonon entry points of include/spk_b200.h are exported by the library and bound by _lib, the ctypes struct has
the field order of spk_ph_t, and the displaced-atom count of spk_vib_t is bound."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ["spk_ph_force_constants", "spk_ph_images", "spk_ph_dynmat", "spk_ph_dos", "spk_ph_thermo",
                "spk_ph_thermo_workspace_bytes"]


def _fields(struct):
    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    body = text[:text.index(f"}} {struct};")].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            decl = re.sub(r"\[\d+\]$", "", decl)
            names += [n.strip().lstrip("*") for n in re.sub(r"^(const\s+)?\w+\*?\s+", "", decl).split(",")]
    return names


def test_phonon_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ENTRY_POINTS:
        assert hasattr(h, name), name
        assert name in _lib.SIGNATURES, name
    assert _lib.SIGNATURES["spk_ph_force_constants"] == [ctypes.POINTER(_lib.PhononParams), _lib.P]
    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    assert f"#define SPK_PH_MAX_IMAGES {_lib.PH_MAX_IMAGES}" in text


def test_phonon_struct_matches_header():
    from schnetpack_b200 import _lib

    assert _fields("spk_ph_t") == [f[0] for f in _lib.PhononParams._fields_]
    assert "n_displaced" in _fields("spk_vib_t")


def test_thermo_workspace_formula():
    from schnetpack_b200 import _lib

    lib = _lib.lib()
    assert lib.spk_ph_thermo_workspace_bytes(1000, 7) == 8 * _lib.PH_THERMO_FIELDS * (7 + 4)
