"""CPU: the C-ABI shared library builds for sm_90a, loads, and exports every symbol include/spk_b200.h declares, and the
binding _lib reads from the header lays the structs out as the C compiler does (no compute calls -- there is no GPU
here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "spk_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(spk_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported():
    from schnetpack_b200 import _lib, build

    path = build.build()
    assert os.path.exists(path)
    h = ctypes.CDLL(path)
    declared = _declared_symbols()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(h, name), f"{name} declared in spk_b200.h but not exported"
    # the ctypes table binds exactly the declared entry points
    assert sorted(_lib.SIGNATURES) == declared
    assert h.spk_version() >= 1
    assert h.spk_graph_workspace_bytes  # callable without a device


def test_struct_layouts_match_the_c_compiler(tmp_path):
    """Every parameter struct _lib reads from the header has the C compiler's size and field offsets: field order, types
    and padding."""
    import shutil
    import subprocess

    from schnetpack_b200 import _lib

    cc = shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spk_b200.h")).read(), flags=re.S)
    assert sorted(_lib.STRUCTS) == sorted(re.findall(r"\}\s*(\w+)\s*;", text))
    expected, prints = {}, []
    for name, struct in _lib.STRUCTS.items():
        expected[name] = ctypes.sizeof(struct)
        prints.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for field, _ in struct._fields_:
            expected[f"{name}.{field}"] = getattr(struct, field).offset
            prints.append(f'printf("{name}.{field} %zu\\n", offsetof({name}, {field}));')
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "spk_b200.h"\nint main(void) {\n'
                   + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "layout")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True, check=True).stdout
    assert {k: int(v) for k, v in (line.split() for line in out.splitlines())} == expected


@pytest.mark.parametrize("header, message", [
    ("int spk_f(long n, spk_stream_t stream);", "unknown type 'long'"),
    ("void spk_f(int n);", "spk_f returns 'void'"),
    ("typedef struct { int16_t n; } spk_s_t;", "unknown type 'int16_t'"),
])
def test_header_reader_refuses_unknown_constructs(header, message):
    from schnetpack_b200 import _lib

    with pytest.raises(ValueError, match=message):
        _lib.read_header(header)


def test_sm100a_sass_present():
    import shutil
    import subprocess

    from schnetpack_b200 import build

    path = build.build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", path], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_cpu_fallback():
    """The product path refuses CPU tensors instead of silently computing elsewhere."""
    import torch

    import schnetpack_b200 as sb
    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import from_spec

    spec, inputs = S.make_config("cfg1")
    model = from_spec(spec, S.init_params(spec, 0))
    x = {k: torch.as_tensor(v) for k, v in inputs.items()}
    x["_positions"] = x["_positions"].float()
    x["_offsets"] = x["_offsets"].float()
    with pytest.raises(RuntimeError, match="CUDA"):
        model(x)


def test_training_mode_is_the_only_way_onto_the_aten_path():
    """train() mode with trainable weights evaluates the differentiable ATen formulas (functional_torch, row f3 --
    tests/test_training_path.py pins it to the reference's weight gradients); the moment the model is in eval() mode, or no
    parameter is trainable, or grad mode is off, the kernels are the only path and CPU tensors raise."""
    import torch

    from schnetpack_b200 import synthetic as S
    from schnetpack_b200.model import from_spec

    spec, inputs = S.make_config("cfg1")
    model = from_spec(spec, S.init_params(spec, 0))
    x = lambda: {k: (torch.as_tensor(v).float() if v.dtype.kind == "f" else torch.as_tensor(v)) for k, v in inputs.items()}  # noqa: E731
    model.train()
    out = model(x())
    assert out["forces"].requires_grad                   # create_graph=self.training: differentiable forces
    with torch.no_grad():
        with pytest.raises(RuntimeError):                # grad mode off (and no forces possible): kernels only
            model.representation(dict(x(), _Rij=torch.zeros((inputs["_idx_i"].shape[0], 3))))
    for p in model.parameters():
        p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(x())
    model.eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        model(x())


def test_product_does_not_import_oracle():
    """Nothing under schnetpack_b200/ may import oracle/ (the oracle is test infrastructure)."""
    import glob

    for f in glob.glob(os.path.join(ROOT, "schnetpack_b200", "**", "*.py"), recursive=True):
        src = open(f).read()
        assert "import oracle" not in src and "from oracle" not in src, f
