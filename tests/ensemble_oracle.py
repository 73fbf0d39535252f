"""fp64 numpy restatement of the reference's ensemble statistics, the checker of csrc/ensemble.cu and of the ensemble
modes of DeviceMD / DeviceLBFGS (paths relative to the reference's src/schnetpack):

  * ``accumulate``: EnsembleCalculator._accumulate_results (md/calculators/ensemble_calculator.py:38-59): mean and the
    unbiased torch.var over the members;
  * ``nn_ensemble``: NNEnsemble.forward (interfaces/batchwise_optimization.py:52-72): mean and the unbiased torch.std;
  * ``uncertainty``: AbsoluteUncertainty / RelativeUncertainty (interfaces/ase_interface.py:340-432) for one structure,
    np.std with ddof = 0, and ``batched_uncertainty`` for a batch, with the force term of an empty system set to 0.
"""
import numpy as np

EPS = 1e-8     # ase_interface.py:402,414,427


def accumulate(stack):
    """{p: [K, ...]} -> {p: mean, p_var: unbiased variance} (ensemble_calculator.py:55-59)"""
    out = {}
    for p, x in stack.items():
        x = np.asarray(x, dtype=np.float64)
        out[p] = x.mean(0)
        out[p + "_var"] = x.var(0, ddof=1)
    return out


def nn_ensemble(stack):
    """{p: [K, ...]} -> (means, stds) with the unbiased std (batchwise_optimization.py:66-70)"""
    means, stds = {}, {}
    for p, x in stack.items():
        x = np.asarray(x, dtype=np.float64)
        means[p], stds[p] = x.mean(0), x.std(0, ddof=1)
    return means, stds


def normalised_weights(energy_weight=0.0, force_weight=1.0, stress_weight=0.0):
    """ase_interface.py:350-358"""
    total = energy_weight + force_weight + stress_weight
    if total == 0:
        raise ValueError("total_weight cannot be zero")
    return energy_weight / total, force_weight / total, stress_weight / total


def uncertainty(energy, forces, stress=None, weights=(0.0, 1.0, 0.0), relative=False):
    """One structure: energy [K], forces [K, n, 3], stress [K, 3, 3] (ase_interface.py:365-432)"""
    we, wf, ws = normalised_weights(*weights)
    u = 0.0
    if we > 0:
        e = np.asarray(energy, dtype=np.float64).reshape(-1)
        sd = np.std(e)
        u += we * (sd / (abs(np.mean(e)) + EPS) if relative else sd)
    if wf > 0:
        f = np.asarray(forces, dtype=np.float64)
        sd = np.linalg.norm(np.std(f, axis=0), axis=1)
        if relative:
            sd = sd / (np.linalg.norm(np.mean(f, axis=0), axis=1) + EPS)
        u += wf * (np.mean(sd) if sd.size else 0.0)       # an empty structure: 0 (the reference's mean would be NaN)
    if ws > 0:
        s = np.asarray(stress, dtype=np.float64)
        sd = np.linalg.norm(np.std(s, axis=0), axis=1)
        if relative:
            sd = sd / (np.linalg.norm(np.mean(s, axis=0), axis=1) + EPS)
        u += ws * np.mean(sd)
    return u


def batched_uncertainty(energy, forces, n_atoms, stress=None, weights=(0.0, 1.0, 0.0), relative=False):
    """energy [K, B], forces [K, N, 3] (systems in order, n_atoms [B]), stress [K, B, 3, 3] -> [B]"""
    ptr = np.concatenate([[0], np.cumsum(n_atoms)]).astype(np.int64)
    out = np.zeros(len(n_atoms))
    for b in range(len(n_atoms)):
        out[b] = uncertainty(None if energy is None else np.asarray(energy)[:, b],
                             np.asarray(forces)[:, ptr[b]:ptr[b + 1]],
                             None if stress is None else np.asarray(stress)[:, b], weights, relative)
    return out


def force_terms(forces, n_atoms, scale=1.0):
    """the per-system sums of spk_ensemble_forces: (sum_i ||std_0(F_i)||, sum_i ||std_0|| / (||mean|| + 1e-8)) of the
    forces x scale, [B, 2]"""
    f = np.asarray(forces, dtype=np.float64) * scale
    sd = np.linalg.norm(f.std(0), axis=1)
    rel = sd / (np.linalg.norm(f.mean(0), axis=1) + EPS)
    ptr = np.concatenate([[0], np.cumsum(n_atoms)]).astype(np.int64)
    return np.array([[sd[ptr[b]:ptr[b + 1]].sum(), rel[ptr[b]:ptr[b + 1]].sum()] for b in range(len(n_atoms))])
