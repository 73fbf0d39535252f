"""CPU: the NEB entry points of include/spk_b200.h are exported by the library and bound by _lib, and the ctypes struct
has the field order of spk_neb_t."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def test_neb_struct_matches_header():
    from schnetpack_b200 import _lib

    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    body = text[:text.index("} spk_neb_t;")].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [n.strip().lstrip("*") for n in re.sub(r"^(const\s+)?\w+\*?\s+", "", decl).split(",")]
    assert names == [f[0] for f in _lib.NEBState._fields_]
