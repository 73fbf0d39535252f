"""CPU: the C-ABI shared library builds for sm_90a, loads, and exports every symbol include/spk_b200.h declares
(no compute calls -- there is no GPU here)."""
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
