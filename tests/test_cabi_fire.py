"""CPU: the FIRE entry points of include/spk_b200.h are exported by the library and bound by _lib, and the ctypes struct
has the field order of spk_fire_t."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fire_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ("spk_fire_workspace_bytes", "spk_fire_forces", "spk_fire_step"):
        assert hasattr(h, name), name
    assert _lib.SIGNATURES["spk_fire_forces"] == [ctypes.POINTER(_lib.FIREState), _lib.P, _lib.P, _lib.P]
    assert _lib.SIGNATURES["spk_fire_step"] == [ctypes.POINTER(_lib.FIREState), _lib.P]
    assert _lib.LAUNCHES["spk_fire_forces"] == 3 and _lib.LAUNCHES["spk_fire_step"] == 2
    ws = _lib.lib().spk_fire_workspace_bytes
    assert ws(0, 1) == 3 * 8 and ws(257, 2) == 3 * 8 * (2 + 2)      # 3 sums per system and per CTA of 256 atoms


def test_fire_struct_matches_header():
    from schnetpack_b200 import _lib

    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    body = text[:text.index("} spk_fire_t;")].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [re.sub(r"\[\d+\]$", "", n.strip().lstrip("*"))
                      for n in re.sub(r"^(const\s+)?\w+\*?\s+", "", decl).split(",")]
    assert names == [f[0] for f in _lib.FIREState._fields_]
    assert _lib.FIREState.mask.size == 9 * ctypes.sizeof(ctypes.c_double)
