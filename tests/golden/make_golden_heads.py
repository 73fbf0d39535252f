"""Regenerate the DipoleMoment / Polarizability fixtures tests/golden/heads_*.npz from the UNMODIFIED reference
(oracle/ref_loader via tests/heads_oracle.py): the model [PairwiseDistances] -> rep -> [Atomwise, Forces, heads...] with
the reference's own head initialisation (torch.manual_seed(HEAD_SEED)), every weight stored, the inputs, and the fp32 and
fp64 outputs including the derivatives d(dipole)/dR [3 or 1, N, 3] and d(polarizability)/dR [9, N, 3] ("d:<key>").

Run from the repository root:  python tests/golden/make_golden_heads.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from make_golden import save_case  # noqa: E402

import heads_oracle as HO  # noqa: E402
from schnetpack_b200 import synthetic as S  # noqa: E402


def main():
    torch.set_grad_enabled(True)
    for name in HO.CASES:
        spec, inputs, heads = HO.case_inputs(name)
        params = S.init_params(spec, HO.REP_SEED)
        model = HO.build_reference(spec, params, heads, torch.float32)
        flat = {k: v.detach().numpy() for k, v in model.state_dict().items()}
        outs = {}
        for tag, dt in (("32", torch.float32), ("64", torch.float64)):
            m = HO.build_reference(spec, params, heads, dt, head_params=flat)
            outs[tag] = HO.run_reference(m, inputs, heads, dt)
        save_case(name, spec, HO.REP_SEED, inputs, outs["32"], outs["64"], params=flat)


if __name__ == "__main__":
    main()
