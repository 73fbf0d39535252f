"""CPU: the vibrational-analysis entry points of include/spk_b200.h are exported by the library and bound by _lib, and
the ctypes struct has the field order of spk_vib_t."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ["spk_vib_displace", "spk_vib_assemble", "spk_vib_finish"]


def test_vibration_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ENTRY_POINTS:
        assert hasattr(h, name), name
        assert _lib.SIGNATURES[name] == [ctypes.POINTER(_lib.VibParams), _lib.P]


def test_vib_struct_matches_header():
    from schnetpack_b200 import _lib

    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    body = text[:text.index("} spk_vib_t;")].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [n.strip().lstrip("*") for n in re.sub(r"^(const\s+)?\w+\*?\s+", "", decl).split(",")]
    assert names == [f[0] for f in _lib.VibParams._fields_]
