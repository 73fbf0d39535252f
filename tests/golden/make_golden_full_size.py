"""Stored checker of tests/test_reference_live.py::test_full_size_parity_against_reference_on_gpu: the reference's own modules
(oracle/ref_loader.py) evaluated in fp64 on the CPU at the full sizes of cfg2, cfg3 and cfg4, params seed 7.  The inputs are
not stored: ``synthetic.make_config`` regenerates them bit for bit from its fixed seeds.

    python tests/golden/make_golden_full_size.py      # needs the reference modules; writes tests/golden/full_size_<cfg>.npz
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader as rl  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402

SEED = 7


def main(cfgs=("cfg2", "cfg3", "cfg4")):
    torch.set_num_threads(os.cpu_count() or 1)
    for cfg in cfgs:
        spec, data = S.make_config(cfg)
        params = S.init_params(spec, seed=SEED)
        ref = rl.evaluate(rl.build_from_spec(spec, params, torch.float64), data, torch.float64,
                          forces=bool(spec.get("forces", True)))
        out = {"seed": np.int64(SEED), "n_atoms": np.int64(data[S.Z].shape[0]), "n_edges": np.int64(data[S.idx_i].shape[0])}
        out.update({"ref64:" + k: v.detach().cpu().numpy().astype(np.float64) for k, v in ref.items() if k in ("energy", "forces")})
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", f"full_size_{cfg}.npz"), **out)
        print(cfg, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(tuple(sys.argv[1:]) or ("cfg2", "cfg3", "cfg4"))
