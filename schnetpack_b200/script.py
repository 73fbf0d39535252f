"""TorchScript deployment of the CUDA path (SURVEY.md section 8 f4).

The reference deploys models with ``torch.jit.script`` (``src/scripts/spkdeploy:16-38``; MD with ``script_model=True``,
``md/calculators/schnetpack_calculator.py:105-107``).  The kernel pipelines of this package are driven from Python
(ctypes over the C ABI), which TorchScript cannot compile -- but it can CALL dispatcher ops.  This module therefore
registers the pipelines as custom ops of the library ``spk_b200`` (``torch.library``; forward + first-order backward, the
tape travels as an extra ``Tensor[]`` output so that nothing is hidden from autograd) and provides TorchScript-compatible
module classes whose ``forward`` is nothing but tensor-dict plumbing around those ops:

    scripted = torch.jit.script(schnetpack_b200.script.to_scriptable(convert_model(reference_model)))
    scripted.save("deployed_model")                      # what spkdeploy writes
    ...
    import schnetpack_b200.script                          # registers the ops (once per process), then
    model = torch.jit.load("deployed_model")               # forces via torch.autograd.grad inside the scripted Forces module

The ops run the same kernels as the eager modules (the op implementation re-creates the eager module around the weight
tensors it is handed, without copying them, and calls the same pipelines).  Loading needs a Python host with this package
imported; a pure-C++ host (the LAMMPS pair style, ``interfaces/lammps/pair_schnetpack.cpp:122-132``) would need the same ops
registered from C++ (``TORCH_LIBRARY``) over the same C ABI -- not provided.
"""
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F_

from . import functional as K
from . import nn as snn
from . import ops, properties, representation
from .model import NeuralNetworkPotential

Tensor = torch.Tensor

__all__ = ["to_scriptable", "ScriptedPotential"]

_LIB = torch.library.Library("spk_b200", "DEF")
_LIB.define("pairwise(Tensor R, Tensor offsets, Tensor idx_i, Tensor idx_j) -> Tensor")
_LIB.define("embedding(Tensor table, Tensor Z) -> Tensor")
_LIB.define("representation(str kind, Tensor r_ij, Tensor x0, Tensor idx_i, Tensor idx_j, Tensor[] weights, int[] iparams, "
            "float[] fparams) -> (Tensor, Tensor, Tensor[])")
_LIB.define("atomwise(Tensor q, Tensor idx_m, Tensor[] weights, int n_mol, int act) -> (Tensor, Tensor, Tensor[])")

_ACTS = {ops.ACT_NONE: None, ops.ACT_SILU: F_.silu, ops.ACT_SSP: snn.shifted_softplus}


# ---------------------------------------------------------------------------------------------- eager modules behind the ops
_MODULES: "dict[tuple, nn.Module]" = {}


def _module_for(kind: str, weights: List[Tensor], ip: List[int], fp: List[float]) -> nn.Module:
    """The eager representation module whose parameters / buffers ARE the given tensors (``load_state_dict(assign=True)``),
    cached on the identity of the weight tensors."""
    key = (kind, tuple(int(v) for v in ip), tuple(float(v) for v in fp), tuple(w.data_ptr() for w in weights))
    mod = _MODULES.get(key)
    if mod is not None:
        return mod
    n_atom_basis, n_interactions, n_rbf, rbf_kind, act, shared, shared_filters, n_filters = ip[:8]
    cutoff, eps = fp[0], fp[1]
    # skeleton on the CPU (tiny); load_state_dict(assign=True) below swaps in the caller's (device) tensors without a copy
    rbf = snn.GaussianRBF(n_rbf, cutoff) if rbf_kind == ops.RBF_GAUSSIAN else snn.BesselRBF(n_rbf, cutoff)
    cut = snn.CosineCutoff(cutoff)
    if kind == "painn":
        mod = representation.PaiNN(n_atom_basis, n_interactions, rbf, cut, activation=_ACTS[act],
                                   shared_interactions=bool(shared), shared_filters=bool(shared_filters), epsilon=eps)
    else:
        mod = representation.SchNet(n_atom_basis, n_interactions, rbf, cut, n_filters=n_filters,
                                    shared_interactions=bool(shared), activation=_ACTS[act])
    keys = list(mod.state_dict().keys())
    if len(keys) != len(weights):
        raise RuntimeError(f"spk_b200::representation: expected {len(keys)} weight tensors, got {len(weights)}")
    mod.load_state_dict({k: w for k, w in zip(keys, weights)}, assign=True)
    mod.eval()
    if len(_MODULES) > 16:
        _MODULES.pop(next(iter(_MODULES)))
    _MODULES[key] = mod
    return mod


def _flatten_painn(saved):
    phi, dphi, geo, tape = saved
    flat = [phi, dphi, geo]
    for hpre, x, mu, (VW, cpre, s) in tape:
        flat += [hpre, x, mu if mu is not None else phi.new_zeros(0), VW, cpre, s]
    return flat


def _unflatten_painn(flat):
    phi, dphi, geo = flat[:3]
    tape = []
    for t in range((len(flat) - 3) // 6):
        hpre, x, mu, VW, cpre, s = flat[3 + 6 * t: 9 + 6 * t]
        tape.append((hpre, x, mu if mu.numel() else None, (VW, cpre, s)))
    return phi, dphi, geo, tape


def _flatten_schnet(saved):
    phi, dphi, geo, tape = saved
    flat = [phi, dphi, geo]
    for item in tape:
        flat += list(item)
    return flat


def _unflatten_schnet(flat):
    phi, dphi, geo = flat[:3]
    return phi, dphi, geo, [tuple(flat[3 + 4 * t: 7 + 4 * t]) for t in range((len(flat) - 3) // 4)]


# ---------------------------------------------------------------------------------------------- op implementations
def _pairwise(R, offsets, idx_i, idx_j):
    with ops.device_of(R):
        return ops.pairwise_fwd(R.detach().contiguous(), idx_i.contiguous(), idx_j.contiguous(),
                                offsets.detach().contiguous())


def _pairwise_ctx(ctx, inputs, output):
    ctx.idx = (inputs[2], inputs[3], inputs[0].shape[0])


def _pairwise_bwd(ctx, g):
    idx_i, idx_j, n = ctx.idx
    with ops.device_of(g):
        graph = ops.get_graph(idx_i, idx_j, n)
        g = g.contiguous()
        return ops.pairwise_bwd(g, graph, 1.0), g, None, None


def _embedding(table, Z):
    with ops.device_of(table):
        return ops.embedding(table.detach().contiguous(), Z)


def _representation(kind, r_ij, x0, idx_i, idx_j, weights, ip, fp):
    mod = _module_for(kind, weights, ip, fp)
    need = bool(ip[8])
    with ops.device_of(r_ij, x0):
        pk = mod._pack()
        r = r_ij.detach().contiguous()
        if kind == "painn":
            graph = ops.get_graph(idx_i, idx_j, x0.shape[0])
            q, mu, saved = K.painn_forward(pk, x0.detach().contiguous(), r, graph, mod._rbf_kind, mod._n_rbf, mod._rbf_p0,
                                           mod._rbf_p1, mod._cutoff_value, mod._act, need)
            return q, mu, (_flatten_painn(saved) if need else [])
        if not need and ops.cfconv_tc_ok(pk.F, pk.NF, mod._n_rbf, r.shape[0]):
            x = K.schnet_forward_fused(pk, x0.detach().contiguous(), r, idx_i, idx_j, mod._rbf_kind, mod._n_rbf, mod._rbf_p0,
                                       mod._rbf_p1, mod._cutoff_value, mod._act)
            return x, x.new_zeros(0), []
        graph = ops.get_graph(idx_i, idx_j, x0.shape[0])
        x, saved = K.schnet_forward(pk, x0.detach().contiguous(), r, graph, mod._rbf_kind, mod._n_rbf, mod._rbf_p0,
                                    mod._rbf_p1, mod._cutoff_value, mod._act, need)
        return x, x.new_zeros(0), (_flatten_schnet(saved) if need else [])


def _representation_ctx(ctx, inputs, output):
    kind, r_ij, x0, idx_i, idx_j, weights, ip, fp = inputs
    ctx.h = (kind, idx_i, idx_j, weights, ip, fp, x0.shape[0], r_ij.shape[0], output[2])


def _representation_bwd(ctx, g_a, g_b, g_tape):
    kind, idx_i, idx_j, weights, ip, fp, n_atoms, n_edges, flat = ctx.h
    if len(flat) == 0:
        raise RuntimeError("spk_b200::representation was run without a tape (r_ij did not require grad)")
    mod = _module_for(kind, weights, ip, fp)
    some = g_a if g_a is not None else g_b
    with ops.device_of(some):
        pk = mod._pack()
        graph = ops.get_graph(idx_i, idx_j, n_atoms)
        if kind == "painn":
            g_q = g_a.contiguous() if g_a is not None else torch.zeros((n_atoms, pk.F), dtype=torch.float32, device=some.device)
            g_mu = g_b.contiguous() if g_b is not None else None
            g_rij = K.painn_backward(pk, _unflatten_painn(flat), graph, mod._n_rbf, mod._act, g_q, g_mu, n_edges)
        else:
            g_rij = K.schnet_backward(pk, _unflatten_schnet(flat), graph, mod._n_rbf, mod._act, g_a.contiguous(), n_edges)
    return None, g_rij, None, None, None, [None] * len(weights), None, None


def _atomwise(q, idx_m, weights, n_mol, act):
    w0, b0, w1, b1 = weights
    with ops.device_of(q):
        l0 = _lin_for(w0, b0)
        hid, hpre = l0.fwd(q.detach().contiguous(), act, save_deriv=True)
        mol_ptr = ops.segment_ptr(idx_m, n_mol)
        y, energy = ops.atomwise_out(hid, w1.detach().reshape(-1).contiguous(), b1.detach().contiguous(), mol_ptr, n_mol)
    return y, energy, [hpre]


_LINS: "dict[tuple, ops.Lin]" = {}


def _lin_for(w, b):
    key = (w.data_ptr(), w._version, b.data_ptr(), b._version)
    lin = _LINS.get(key)
    if lin is None:
        if len(_LINS) > 16:
            _LINS.pop(next(iter(_LINS)))
        lin = _LINS[key] = ops.Lin(w, b)
    return lin


def _atomwise_ctx(ctx, inputs, output):
    q, idx_m, weights, n_mol, act = inputs
    ctx.h = (idx_m, weights, q.shape[0], output[2][0])


def _atomwise_bwd(ctx, g_y, g_e, g_tape):
    idx_m, weights, n_atoms, hpre = ctx.h
    w0, b0, w1, b1 = weights
    w1f = w1.detach().reshape(-1).contiguous()
    with ops.device_of(hpre):
        g_hid = None
        if g_e is not None:
            g_hid = ops.atomwise_out_bwd(g_e.contiguous(), idx_m, w1f, n_atoms, w1f.shape[0])
        if g_y is not None:
            extra = g_y.contiguous()[:, None] * w1f[None, :]
            g_hid = extra if g_hid is None else g_hid + extra
        g_q = _lin_for(w0, b0).bwd(g_hid.contiguous(), a_pre=hpre, a_act=ops.ACT_GIVEN)
    return g_q, None, [None] * 4, None, None


_LIB.impl("pairwise", _pairwise, "CompositeExplicitAutograd")
_LIB.impl("embedding", _embedding, "CompositeExplicitAutograd")
_LIB.impl("representation", _representation, "CompositeExplicitAutograd")
_LIB.impl("atomwise", _atomwise, "CompositeExplicitAutograd")
torch.library.register_autograd("spk_b200::pairwise", _pairwise_bwd, setup_context=_pairwise_ctx)
torch.library.register_autograd("spk_b200::representation", _representation_bwd, setup_context=_representation_ctx)
torch.library.register_autograd("spk_b200::atomwise", _atomwise_bwd, setup_context=_atomwise_ctx)


# ---------------------------------------------------------------------------------------------- TorchScript-compatible modules
class ScriptPairwiseDistances(nn.Module):
    """atomistic/distances.py:9-26 on ``spk_b200::pairwise``."""

    def forward(self, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
        inputs["_Rij"] = torch.ops.spk_b200.pairwise(inputs["_positions"], inputs["_offsets"], inputs["_idx_i"],
                                                     inputs["_idx_j"])
        return inputs


class ScriptRepresentation(nn.Module):
    """PaiNN / SchNet (representation/painn.py:207-256, schnet.py:147-173) on ``spk_b200::representation``; weights are held
    as a flat list in ``state_dict`` order of the eager module."""

    def __init__(self, rep: nn.Module):
        super().__init__()
        if not isinstance(rep, (representation.PaiNN, representation.SchNet)):
            raise NotImplementedError(f"to_scriptable: {type(rep).__name__} has no TorchScript deployment (PaiNN and "
                                      "SchNet only)")
        self.kind = "painn" if isinstance(rep, representation.PaiNN) else "schnet"
        if not isinstance(rep.embedding, nn.Embedding) or len(rep.electronic_embeddings) > 0:
            raise NotImplementedError("to_scriptable: plain nn.Embedding representations")
        self.weights = nn.ParameterList([nn.Parameter(v.detach(), requires_grad=False) for v in rep.state_dict().values()])
        self.emb_index = list(rep.state_dict().keys()).index("embedding.weight")
        shared = len(rep.interactions) > 1 and rep.interactions[0] is rep.interactions[1]
        self.iparams = [int(rep.n_atom_basis), len(rep.interactions), int(rep.radial_basis.n_rbf), int(rep.radial_basis.kind),
                        int(snn.activation_code(rep.activation)), int(shared), int(getattr(rep, "share_filters", False)),
                        int(getattr(rep, "n_filters", rep.n_atom_basis))]
        eps = float(rep.mixing[0].epsilon) if self.kind == "painn" else 0.0
        self.fparams = [float(rep.cutoff_fn.value()), eps]
        self.cutoff = rep.cutoff                                  # read by spkdeploy:38
        self.n_atom_basis = int(rep.n_atom_basis)

    def forward(self, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
        r_ij = inputs["_Rij"]
        ws: List[Tensor] = []
        for p in self.weights:
            ws.append(p)
        x0 = torch.ops.spk_b200.embedding(ws[self.emb_index], inputs["_atomic_numbers"])
        ip: List[int] = []
        for v in self.iparams:
            ip.append(v)
        ip.append(int(r_ij.requires_grad))
        a, b, tape = torch.ops.spk_b200.representation(self.kind, r_ij, x0, inputs["_idx_i"], inputs["_idx_j"], ws, ip,
                                                       self.fparams)
        inputs["scalar_representation"] = a
        if self.kind == "painn":
            inputs["vector_representation"] = b
        return inputs


class ScriptAtomwise(nn.Module):
    """atomistic/atomwise.py:69-88 (n_out = 1, two layers, sum / avg aggregation) on ``spk_b200::atomwise``."""

    def __init__(self, head: nn.Module):
        super().__init__()
        if head.n_out != 1 or len(head.outnet) != 2 or head.aggregation_mode not in ("sum", "avg"):
            raise NotImplementedError("to_scriptable: Atomwise(n_out=1, n_layers=2, aggregation_mode in {sum, avg})")
        l0, l1 = head.outnet[0], head.outnet[1]
        self.weights = nn.ParameterList([nn.Parameter(t.detach(), requires_grad=False)
                                         for t in (l0.weight, l0.bias, l1.weight, l1.bias)])
        self.act = int(snn.activation_code(head.activation))
        self.output_key = head.output_key
        self.per_atom_output_key: Optional[str] = head.per_atom_output_key
        self.avg = head.aggregation_mode == "avg"
        self.model_outputs: List[str] = list(head.model_outputs)

    def forward(self, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
        ws: List[Tensor] = []
        for p in self.weights:
            ws.append(p)
        n_mol = inputs["_n_atoms"].shape[0]
        y, e, tape = torch.ops.spk_b200.atomwise(inputs["scalar_representation"], inputs["_idx_m"], ws, n_mol, self.act)
        key = self.per_atom_output_key
        if key is not None:
            inputs[key] = y.unsqueeze(-1)
        if self.avg:
            e = e / inputs["_n_atoms"]
        inputs[self.output_key] = e
        return inputs


class ScriptForces(nn.Module):
    """atomistic/response.py:18-92 (forces only): -dE/dR through torch.autograd.grad, as the reference does in TorchScript."""

    def __init__(self, mod: nn.Module):
        super().__init__()
        if mod.calc_stress:
            raise NotImplementedError("to_scriptable: Forces(calc_stress=False)")
        self.energy_key = mod.energy_key
        self.force_key = mod.force_key
        self.model_outputs: List[str] = [mod.force_key]
        self.required_derivatives: List[str] = [properties.R]

    def forward(self, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
        Epred = inputs[self.energy_key]
        go: List[Optional[Tensor]] = [torch.ones_like(Epred)]
        grads = torch.autograd.grad([Epred], [inputs["_positions"]], grad_outputs=go, create_graph=False)
        dEdR = grads[0]
        if dEdR is None:
            dEdR = torch.zeros_like(inputs["_positions"])
        inputs[self.force_key] = -dEdR
        return inputs


class ScriptedPotential(nn.Module):
    """model/base.py:132-190 (NeuralNetworkPotential.forward) over the scriptable modules."""

    required_derivatives: List[str]          # class-level annotations: the lists may be empty (energy-only models)
    model_outputs: List[str]

    def __init__(self, input_modules, rep, output_modules, postprocessors, required_derivatives, model_outputs,
                 do_postprocessing: bool):
        super().__init__()
        self.input_modules = nn.ModuleList(input_modules)
        self.representation = rep
        self.output_modules = nn.ModuleList(output_modules)
        self.postprocessors = nn.ModuleList(postprocessors)
        self.required_derivatives: List[str] = list(required_derivatives)
        self.model_outputs: List[str] = list(model_outputs)
        self.do_postprocessing = do_postprocessing

    def forward(self, inputs: Dict[str, Tensor]) -> Dict[str, Tensor]:
        for p in self.required_derivatives:
            if p in inputs:
                inputs[p].requires_grad_()
        for m in self.input_modules:
            inputs = m(inputs)
        inputs = self.representation(inputs)
        for m in self.output_modules:
            inputs = m(inputs)
        if self.do_postprocessing:
            for pp in self.postprocessors:
                inputs = pp(inputs)
        results: Dict[str, Tensor] = {}
        for k in self.model_outputs:
            results[k] = inputs[k]
        return results


def to_scriptable(model: NeuralNetworkPotential) -> ScriptedPotential:
    """TorchScript-compatible twin of a CUDA ``NeuralNetworkPotential`` (``convert_model`` output or ``from_spec``): same
    weights (shared storage), ``torch.jit.script`` -able, ``save`` / ``load`` -able."""
    ins = []
    for m in model.input_modules:
        if type(m).__name__ != "PairwiseDistances":
            raise NotImplementedError(f"to_scriptable: input module {type(m).__name__}")
        ins.append(ScriptPairwiseDistances())
    outs = []
    for m in model.output_modules:
        n = type(m).__name__
        if n == "Atomwise":
            outs.append(ScriptAtomwise(m))
        elif n == "Forces":
            outs.append(ScriptForces(m))
        elif n in ("DipoleMoment", "Polarizability", "ZBLRepulsionEnergy", "EnergyCoulomb", "EnergyEwald",
                   "EnergyPME", "Aggregation"):
            raise NotImplementedError(f"to_scriptable: {n} has no TorchScript twin (its kernels run through "
                                      "torch.autograd.Function); evaluate the model in Python")
        else:
            outs.append(m)                         # other heads must be scriptable themselves (as in the reference)
    return ScriptedPotential(ins, ScriptRepresentation(model.representation), outs, list(model.postprocessors),
                             model.required_derivatives, model.model_outputs, bool(model.do_postprocessing)).eval()
