"""Model ensembles on the kernels: K independently trained members run on the same inputs, their outputs are stacked into
slots [K, ...], and the statistics over the members come from ``csrc/ensemble.cu`` (fp64, two passes, fixed order,
bitwise reproducible).

  * ``NNEnsemble`` mirrors interfaces/batchwise_optimization.py:36-72: ``forward(inputs) -> (means, stds)`` with the
    unbiased std (torch.std).
  * ``AbsoluteUncertainty`` / ``RelativeUncertainty`` mirror interfaces/ase_interface.py:340-432 (np.std, ddof = 0),
    batched: they take the stacked predictions of a whole batch and its system layout and return [B] fp64.
  * ``md.DeviceMD`` and ``relax.DeviceLBFGS`` take a list of >= 2 members and run the same statistics inside their
    captured step (``md._CapturedEvaluation``).

The ddof of each API is the reference's: the ``{p}_var`` of the MD calculator (ensemble_calculator.py:57-59) and the std of
``NNEnsemble`` are unbiased (ddof = 1), the ASE uncertainties use ddof = 0.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _lib, ops
from . import properties as P

__all__ = ["NNEnsemble", "AbsoluteUncertainty", "RelativeUncertainty", "ensemble_moments", "ensemble_forces",
           "members_of"]

Tensor = torch.Tensor


def members_of(model) -> Optional[List[nn.Module]]:
    """The members of an ensemble given as a list, tuple or ``nn.ModuleList`` (None for a single module).  Fewer than two
    members raise ``ValueError``."""
    if isinstance(model, nn.Module) and not isinstance(model, nn.ModuleList):
        return None
    members = list(model)
    if len(members) < 2:
        raise ValueError(f"an ensemble needs at least two members, got {len(members)}")
    for m in members:
        if not isinstance(m, nn.Module):
            raise TypeError(f"ensemble members must be torch.nn.Module, got {type(m).__name__}")
    return members


def _stacked(x: Tensor, name: str) -> Tensor:
    if not x.is_cuda or x.dtype != torch.float32 or not x.is_contiguous():
        raise TypeError(f"ensemble: '{name}' must be a contiguous float32 CUDA tensor [K, ...]")
    if x.dim() < 1 or x.shape[0] < 1:
        raise ValueError(f"ensemble: '{name}' of shape {tuple(x.shape)} has no member axis")
    return x


def _buffer(t: Optional[Tensor], numel: int, dtype, name: str, at_least: bool = False) -> Optional[Tensor]:
    """``t`` (if given) as a buffer the kernels may read or write ``numel`` elements of: contiguous, on the device, of
    ``dtype``, with exactly (``at_least``: at least) that many elements"""
    if t is None:
        return None
    if not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise TypeError(f"ensemble: '{name}' must be a contiguous {dtype} CUDA tensor")
    if t.numel() < numel or (not at_least and t.numel() != numel):
        raise ValueError(f"ensemble: '{name}' holds {t.numel()} elements, {'at least ' if at_least else ''}{numel} "
                         "needed")
    return t


def ensemble_moments(x: Tensor, ddof: int = 1, mean_scale: float = 1.0, spread_scale: float = 1.0, var: bool = True,
                     std: bool = False, out_mean: Optional[Tensor] = None, out_var: Optional[Tensor] = None,
                     out_std: Optional[Tensor] = None) -> Tuple[Tensor, Optional[Tensor], Optional[Tensor]]:
    """Element-wise mean (x ``mean_scale``), variance with ``ddof`` and std (each x ``spread_scale``) over the first axis
    of the stacked member outputs ``x`` [K, ...] fp32; results are fp32 [...]."""
    x = _stacked(x, "x")
    shape, K = x.shape[1:], int(x.shape[0])
    n = x.numel() // K
    mean = _buffer(out_mean, n, torch.float32, "out_mean")
    if mean is None:
        mean = torch.empty(shape, dtype=torch.float32, device=x.device)
    v = _buffer(out_var, n, torch.float32, "out_var") if out_var is not None else (torch.empty_like(mean) if var else None)
    s = _buffer(out_std, n, torch.float32, "out_std") if out_std is not None else (torch.empty_like(mean) if std else None)
    _lib.call("spk_ensemble_moments", ops._p(x), K, n, int(ddof), float(mean_scale), float(spread_scale), ops._p(mean),
              ops._p(v), ops._p(s), ops._stream())
    return mean, v, s


def ensemble_forces(forces: Tensor, idx_m: Optional[Tensor] = None, sys_ptr: Optional[Tensor] = None, n_sys: int = 0,
                    mean_scale: float = 1.0, spread_scale: float = 1.0, var: bool = True, terms: bool = False,
                    out_mean: Optional[Tensor] = None, out_var: Optional[Tensor] = None,
                    out_terms: Optional[Tensor] = None, workspace: Optional[Tensor] = None):
    """Statistics of stacked forces [K, N, 3]: the mean (x ``mean_scale``) and unbiased per-component variance (x
    ``spread_scale``), and with ``terms`` the per-system sums [n_sys, 2] fp64 of ||std_0(F_i)|| and ||std_0(F_i)|| /
    (||mean(F_i)|| + 1e-8) of the forces x ``spread_scale`` (systems: ``idx_m`` sorted, ``sys_ptr`` its segment
    pointer)."""
    f = _stacked(forces, "forces")
    if f.dim() != 3 or f.shape[2] != 3:
        raise ValueError(f"ensemble_forces: forces must be [K, N, 3], got {tuple(f.shape)}")
    K, n, n_sys = int(f.shape[0]), int(f.shape[1]), int(n_sys)
    dev = f.device
    mean = _buffer(out_mean, 3 * n, torch.float32, "out_mean")
    if mean is None:
        mean = torch.empty(f.shape[1:], dtype=torch.float32, device=dev)
    v = _buffer(out_var, 3 * n, torch.float32, "out_var") if out_var is not None else (torch.empty_like(mean) if var
                                                                                     else None)
    t = ws = None
    if terms:
        if n_sys < 1 or idx_m is None or sys_ptr is None:
            raise ValueError("ensemble_forces: per-system terms need idx_m, sys_ptr and n_sys >= 1")
        _buffer(idx_m, n, torch.int64, "idx_m")
        _buffer(sys_ptr, n_sys + 1, torch.int32, "sys_ptr")
        t = _buffer(out_terms, 2 * n_sys, torch.float64, "out_terms")
        if t is None:
            t = torch.empty(n_sys, 2, dtype=torch.float64, device=dev)
        nbytes = int(_lib.lib().spk_ensemble_workspace_bytes(n, n_sys))
        ws = _buffer(workspace, nbytes, torch.uint8, "workspace", at_least=True)
        if ws is None:
            ws = ensemble_workspace(n, n_sys, dev)
    _lib.call("spk_ensemble_forces", ops._p(f), K, ops._p(idx_m), ops._p(sys_ptr), n, int(n_sys), float(mean_scale),
              float(spread_scale), ops._p(mean), ops._p(v), ops._p(t), ops._p(ws), 0 if ws is None else ws.numel(),
              ops._stream(), launches=(1 if n else 0) + (1 if terms else 0))
    return mean, v, t


def ensemble_workspace(n_atoms: int, n_sys: int, device) -> Tensor:
    nbytes = int(_lib.lib().spk_ensemble_workspace_bytes(int(n_atoms), int(n_sys)))
    return torch.empty(max(nbytes, 8), dtype=torch.uint8, device=device)


class NNEnsemble(nn.Module):
    """interfaces/batchwise_optimization.py:36-72 on the kernels: every member runs on the same inputs (a shallow copy of
    the dict per member, so one member's in-place additions do not reach the next; the reference deep-copies), its
    outputs in ``properties`` are copied into slot k before the next member runs, and ``forward`` returns (means, stds)
    with the unbiased std.  Capturable by ``GraphedPotential``."""

    def __init__(self, models, properties: List[str]):
        super().__init__()
        self.models = models if isinstance(models, nn.ModuleList) else nn.ModuleList(members_of(models))
        members_of(self.models)
        if isinstance(properties, str):
            properties = [properties]
        self.properties = list(properties)

    def forward(self, inputs: Dict[str, Tensor]) -> Tuple[Dict[str, Tensor], Dict[str, Tensor]]:
        K = len(self.models)
        stacks: Dict[str, Tensor] = {}
        for k, model in enumerate(self.models):
            out = model(dict(inputs))
            for p in self.properties:
                v = out[p].detach()
                if k == 0:
                    stacks[p] = torch.empty((K,) + tuple(v.shape), dtype=torch.float32, device=v.device)
                elif tuple(v.shape) != tuple(stacks[p].shape[1:]):
                    raise ValueError(f"NNEnsemble: member {k} predicts '{p}' of shape {tuple(v.shape)}, member 0 "
                                     f"{tuple(stacks[p].shape[1:])}")
                stacks[p][k].copy_(v)
        means, stds = {}, {}
        for p, x in stacks.items():
            means[p], _, stds[p] = ensemble_moments(x, ddof=1, var=False, std=True)
        return means, stds


class Uncertainty:
    """interfaces/ase_interface.py:340-363: keys and weights, normalised to sum 1; a zero total raises ``ValueError``.
    Called on the stacked predictions of a batch ({key: [K, ...]}: energies [K, B], forces [K, N, 3], stress
    [K, B, 3, 3]) and its systems (``idx_m`` [N] sorted, ``n_sys`` = B), it returns [B] fp64: for B = 1 the reference's
    scalar.  A system without atoms gets a force term of 0 (the reference's np.mean over no atoms would be NaN)."""

    relative = False

    def __init__(self, energy_key: str = P.energy, force_key: str = P.forces, stress_key: str = P.stress,
                 energy_weight: float = 0.0, force_weight: float = 1.0, stress_weight: float = 0.0):
        self.energy_key = energy_key
        self.force_key = force_key
        self.stress_key = stress_key
        total_weight = energy_weight + force_weight + stress_weight
        if total_weight == 0:
            raise ValueError("total_weight cannot be zero")
        self.energy_weight = energy_weight / total_weight
        self.force_weight = force_weight / total_weight
        self.stress_weight = stress_weight / total_weight

    def __call__(self, predictions: Dict[str, Tensor], idx_m: Tensor, n_sys: int) -> Tensor:
        n_sys = int(n_sys)
        if n_sys < 1:
            raise ValueError(f"{type(self).__name__}: n_sys must be >= 1, got {n_sys}")
        idx_m = ops.i64(idx_m, "_idx_m")
        used = [(k, w) for k, w in ((self.energy_key, self.energy_weight), (self.force_key, self.force_weight),
                                    (self.stress_key, self.stress_weight)) if w > 0]
        for k, w in used:
            if k not in predictions:
                raise KeyError(f"{type(self).__name__}: the predictions hold no '{k}' (weight {w})")
        members = {int(predictions[k].shape[0]) for k, _ in used}
        if len(members) > 1:
            raise ValueError(f"{type(self).__name__}: the predictions stack different member counts {sorted(members)}")
        if self.force_weight > 0 and predictions[self.force_key].dim() == 3 \
                and idx_m.numel() != predictions[self.force_key].shape[1]:
            raise ValueError(f"{type(self).__name__}: idx_m has {idx_m.numel()} entries for "
                             f"{predictions[self.force_key].shape[1]} atoms")
        if idx_m.numel() and not torch.cuda.is_current_stream_capturing():   # one host read: the layout comes from outside
            if bool((idx_m[1:] < idx_m[:-1]).any()) or int(idx_m[0]) < 0 or int(idx_m[-1]) >= n_sys:
                raise ValueError(f"{type(self).__name__}: idx_m must be sorted with values in [0, {n_sys})")
        sys_ptr = ops.segment_ptr(idx_m, n_sys)
        sums = None
        if self.force_weight > 0:
            _, _, sums = ensemble_forces(predictions[self.force_key], idx_m, sys_ptr, n_sys, var=False, terms=True)
        out = torch.empty(n_sys, dtype=torch.float64, device=idx_m.device)
        self.combine(predictions.get(self.energy_key), sums, sys_ptr, predictions.get(self.stress_key), out)
        return out

    def combine(self, energy: Optional[Tensor], force_sums: Optional[Tensor], sys_ptr: Tensor,
                stress: Optional[Tensor], out: Optional[Tensor], energy_scale: float = 1.0, stress_scale: float = 1.0,
                out_f32: Optional[Tensor] = None):
        """the weighted terms into ``out`` [B] fp64 and / or ``out_f32`` [B], given the per-system force sums of
        ``ensemble_forces`` (of the forces already scaled) and the energies and stress scaled here"""
        if out is None and out_f32 is None:
            raise ValueError(f"{type(self).__name__}: no output buffer")
        n_sys = (out if out is not None else out_f32).numel()
        _buffer(out, n_sys, torch.float64, "out")
        _buffer(out_f32, n_sys, torch.float32, "out_f32")
        members = set()
        for name, x, w in (("energy", energy, self.energy_weight), ("stress", stress, self.stress_weight)):
            if w > 0:
                if x is None:
                    raise KeyError(f"{type(self).__name__}: the predictions hold no {name} (weight {w})")
                _stacked(x, name)
                if x.numel() != int(x.shape[0]) * n_sys * (9 if name == "stress" else 1):
                    raise ValueError(f"{type(self).__name__}: {name} of shape {tuple(x.shape)} for {n_sys} systems")
                members.add(int(x.shape[0]))
        if len(members) > 1:
            raise ValueError(f"{type(self).__name__}: energy and stress stack different member counts")
        K = members.pop() if members else 1
        if self.force_weight > 0:
            if force_sums is None:
                raise ValueError(f"{type(self).__name__}: the force term needs the per-system force sums")
            _buffer(force_sums, 2 * n_sys, torch.float64, "force_sums")
            _buffer(sys_ptr, n_sys + 1, torch.int32, "sys_ptr")
        _lib.call("spk_ensemble_uncertainty", ops._p(energy if self.energy_weight > 0 else None), float(energy_scale),
                  ops._p(force_sums), ops._p(sys_ptr), ops._p(stress if self.stress_weight > 0 else None),
                  float(stress_scale), K, n_sys, 1 if self.relative else 0, self.energy_weight, self.force_weight,
                  self.stress_weight, ops._p(out), ops._p(out_f32), ops._stream())


class AbsoluteUncertainty(Uncertainty):
    """w_E std(E) + w_F mean_i ||std(F_i)|| + w_S mean_rows ||std(sigma_row)|| per system (ase_interface.py:365-391)"""


class RelativeUncertainty(Uncertainty):
    """as ``AbsoluteUncertainty`` with every std over (||mean|| + 1e-8) before averaging (ase_interface.py:394-432)"""

    relative = True
