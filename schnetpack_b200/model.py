"""Minimal mirror of the boundary caller ``schnetpack.model.NeuralNetworkPotential``
(/root/reference/src/schnetpack/model/base.py:16-190) so that the CUDA modules can be assembled and driven exactly
like the reference's (input modules -> representation -> output modules -> postprocessors) on a box where the
reference package is absent, plus ``convert_model`` which swaps the hot-path modules of an already-loaded reference
model for their CUDA counterparts (identical ``state_dict`` keys)."""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import atomistic, representation
from . import nn as snn
from . import ops
from . import properties

__all__ = ["AtomisticModel", "NeuralNetworkPotential", "convert_model"]


class AtomisticModel(nn.Module):
    """model/base.py:16-129."""

    def __init__(self, postprocessors: Optional[List[nn.Module]] = None, input_dtype_str: str = "float32",
                 do_postprocessing: bool = True):
        super().__init__()
        self.input_dtype_str = input_dtype_str
        self.do_postprocessing = do_postprocessing
        self.postprocessors = nn.ModuleList(postprocessors)
        self.required_derivatives: Optional[List[str]] = None
        self.model_outputs: Optional[List[str]] = None

    def collect_derivatives(self) -> List[str]:
        self.required_derivatives = None
        required_derivatives = set()
        for m in self.modules():
            if hasattr(m, "required_derivatives") and m.required_derivatives is not None:
                required_derivatives.update(m.required_derivatives)
        self.required_derivatives = list(required_derivatives)
        return self.required_derivatives

    def collect_outputs(self) -> List[str]:
        self.model_outputs = None
        model_outputs = set()
        for m in self.modules():
            if hasattr(m, "model_outputs") and m.model_outputs is not None:
                model_outputs.update(m.model_outputs)
        self.model_outputs = list(model_outputs)
        return self.model_outputs

    def initialize_derivatives(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        for p in self.required_derivatives:
            if p in inputs.keys():
                inputs[p].requires_grad_()
        return inputs

    def postprocess(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.do_postprocessing:
            for pp in self.postprocessors:
                inputs = pp(inputs)
        return inputs

    def extract_outputs(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        return {k: inputs[k] for k in self.model_outputs}


class NeuralNetworkPotential(AtomisticModel):
    """model/base.py:132-190."""

    def __init__(self, representation: nn.Module, input_modules: List[nn.Module] = None,
                 output_modules: List[nn.Module] = None, postprocessors: Optional[List[nn.Module]] = None,
                 input_dtype_str: str = "float32", do_postprocessing: bool = True):
        super().__init__(input_dtype_str=input_dtype_str, postprocessors=postprocessors,
                         do_postprocessing=do_postprocessing)
        self.representation = representation
        self.input_modules = nn.ModuleList(input_modules)
        self.output_modules = nn.ModuleList(output_modules)
        atomistic.pair_terms.check_short_range_cutoff(representation, self.input_modules)
        atomistic.pair_terms.link_charges(self.output_modules)
        self.collect_derivatives()
        self.collect_outputs()

    # set by ``convert_model`` for models that arrive in double precision (spkmd loads every model as fp64 first,
    # md/calculators/schnetpack_calculator.py:98): floating inputs are cast to fp32 on entry, results back on exit
    cast_inputs: bool = False

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        out_dtype = None
        if self.cast_inputs:
            for k, v in list(inputs.items()):
                if v.is_floating_point() and v.dtype != torch.float32 and k != properties.virial:
                    out_dtype = v.dtype
                    inputs[k] = v.to(torch.float32)
        inputs = self.initialize_derivatives(inputs)
        for m in self.input_modules:
            inputs = m(inputs)
        inputs = self.representation(inputs)
        for m in self.output_modules:
            inputs = m(inputs)
        inputs = self.postprocess(inputs)
        out = self.extract_outputs(inputs)
        if out_dtype is not None:
            out = {k: (v.to(out_dtype) if v.is_floating_point() else v) for k, v in out.items()}
        return out


# --------------------------------------------------------------------------------------------------------- conversion
def _convert_rbf(rb):
    name = type(rb).__name__
    if name == "GaussianRBF":
        out = snn.GaussianRBF(rb.n_rbf, 1.0, trainable=isinstance(rb.widths, nn.Parameter))
    elif name == "BesselRBF":
        out = snn.BesselRBF(rb.n_rbf, 1.0)
    else:
        raise NotImplementedError(f"radial basis {name} has no CUDA kernel")
    out.load_state_dict(rb.state_dict())
    return out


def _convert_representation(rep):
    name = type(rep).__name__
    rbf = _convert_rbf(rep.radial_basis)
    cut = snn.CosineCutoff(float(rep.cutoff_fn.cutoff))
    if type(rep.cutoff_fn).__name__ != "CosineCutoff":
        raise NotImplementedError(f"cutoff {type(rep.cutoff_fn).__name__} has no CUDA kernel")
    emb = rep.embedding if not isinstance(rep.embedding, nn.Embedding) else None
    eemb = list(rep.electronic_embeddings) if len(getattr(rep, "electronic_embeddings", [])) else None
    if name == "PaiNN":
        shared = len(rep.interactions) > 1 and rep.interactions[0] is rep.interactions[1]
        act = rep.interactions[0].interatomic_context_net[0].activation
        new = representation.PaiNN(rep.n_atom_basis, rep.n_interactions, rbf, cut, activation=_map_act(act),
                                   shared_interactions=shared, shared_filters=rep.share_filters,
                                   epsilon=rep.mixing[0].epsilon, nuclear_embedding=emb, electronic_embeddings=eemb)
    elif name == "SchNet":
        shared = len(rep.interactions) > 1 and rep.interactions[0] is rep.interactions[1]
        act = rep.interactions[0].f2out[0].activation
        new = representation.SchNet(rep.n_atom_basis, len(rep.interactions), rbf, cut, n_filters=rep.n_filters,
                                    shared_interactions=shared, activation=_map_act(act), nuclear_embedding=emb,
                                    electronic_embeddings=eemb)
    elif name == "SO3net":
        shared = len(rep.so3convs) > 1 and rep.so3convs[0] is rep.so3convs[1]
        new = representation.SO3net(rep.n_atom_basis, rep.n_interactions, int(rep.lmax), rbf, cut,
                                    shared_interactions=shared,
                                    return_vector_representation=rep.return_vector_representation,
                                    activation=rep.activation, nuclear_embedding=emb, electronic_embeddings=eemb)
    else:
        raise NotImplementedError(f"representation {name} is outside the CUDA hot path")
    new.load_state_dict(rep.state_dict())
    return new


def _map_act(act):
    import torch.nn.functional as F
    code = snn.activation_code(act)
    return {0: None, 1: F.silu, 2: snn.shifted_softplus}[code]


def _gated_layout(outnet):
    """(n_hidden as a list of block output widths, activation) of a reference gated equivariant MLP"""
    blocks = list(outnet)
    return [b.n_sout for b in blocks[:-1]], _map_act(blocks[0].scalar_net[0].activation)


def _convert_head(m):
    n = type(m).__name__
    if n == "Polarizability" or m.use_vector_representation:
        hidden, act = _gated_layout(m.outnet)
        for b in m.outnet:
            if b.n_hidden != b.n_sin:
                raise NotImplementedError(f"{n}: gating widths other than the block input width")
    else:
        hidden, act = [l.out_features for l in list(m.outnet)[:-1]], _map_act(m.outnet[0].activation)
    n_in = m.outnet[0].n_sin if (n == "Polarizability" or m.use_vector_representation) else m.outnet[0].in_features
    kw = dict(n_in=n_in, n_hidden=hidden, n_layers=len(m.outnet), activation=act)
    if n == "Polarizability":
        new = atomistic.Polarizability(**kw, polarizability_key=m.polarizability_key)
    else:
        new = atomistic.DipoleMoment(**kw, predict_magnitude=m.predict_magnitude, return_charges=m.return_charges,
                                     dipole_key=m.dipole_key, charges_key=m.charges_key,
                                     correct_charges=m.correct_charges,
                                     use_vector_representation=m.use_vector_representation)
    new.load_state_dict(m.state_dict())
    return new


def _convert_cutoff_fn(cf):
    if cf is None:
        return None
    if type(cf).__name__ != "CosineCutoff":
        raise NotImplementedError(f"cutoff {type(cf).__name__} of a pair term has no CUDA kernel")
    return snn.CosineCutoff(float(cf.cutoff))


def _convert_pair_term(m):
    """ZBLRepulsionEnergy / EnergyCoulomb (with its potential and switch) -> the kernel modules, state_dict copied."""
    if type(m).__name__ == "ZBLRepulsionEnergy":
        new = atomistic.ZBLRepulsionEnergy(1.0, 1.0, m.output_key, cutoff_fn=_convert_cutoff_fn(m.cutoff_fn))
        for name in ("a_pow", "a_div", "coefficients", "exponents"):
            getattr(new, name).requires_grad_(getattr(m, name).requires_grad)
    else:
        pot = m.coulomb_potential
        pn = type(pot).__name__
        if pn == "CoulombPotential":
            new_pot = atomistic.CoulombPotential()
        elif pn == "DampedCoulombPotential" and type(pot.switch_fn).__name__ == "SwitchFunction":
            new_pot = atomistic.DampedCoulombPotential(snn.SwitchFunction(float(pot.switch_fn.switch_on),
                                                                          float(pot.switch_fn.switch_off)))
        else:
            raise NotImplementedError(f"EnergyCoulomb potential {pn} has no CUDA kernel")
        new = atomistic.EnergyCoulomb(1.0, 1.0, new_pot, m.output_key, charges_key=m.charges_key,
                                      use_neighbors_lr=m.use_neighbors_lr,
                                      cutoff=float(m.cutoff) if m.cutoff is not None else None)
    new.load_state_dict(m.state_dict())
    return new


def _convert_ewald(m):
    """EnergyEwald (screening_fn None or SwitchFunction) -> the kernel module, state_dict (ke, alpha, kvecs) copied."""
    sw = m.screening_fn
    if sw is not None and type(sw).__name__ != "SwitchFunction":
        raise NotImplementedError(f"EnergyEwald screening_fn {type(sw).__name__} has no CUDA kernel")
    new_sw = snn.SwitchFunction(float(sw.switch_on), float(sw.switch_off)) if sw is not None else None
    new = atomistic.EnergyEwald(float(m.alpha), int(m.k_max), 1.0, 1.0, m.output_key, charges_key=m.charges_key,
                                use_neighbors_lr=m.use_neighbors_lr, screening_fn=new_sw)
    new.load_state_dict(m.state_dict())
    return new


def convert_model(model: nn.Module) -> NeuralNetworkPotential:
    """Build a CUDA ``NeuralNetworkPotential`` from a loaded reference model (duck-typed on class names; weights are
    copied through ``state_dict`` whose keys are identical).  ``Atomwise`` (n_out=1, n_layers=2), ``Forces``,
    ``DipoleMoment`` and ``Polarizability`` heads, the pair terms ``ZBLRepulsionEnergy`` (cutoff_fn None or CosineCutoff)
    and ``EnergyCoulomb`` (CoulombPotential or DampedCoulombPotential with a SwitchFunction), ``EnergyEwald``
    (screening_fn None or SwitchFunction), ``Aggregation`` and the input modules ``PairwiseDistances`` /
    ``FilterShortRange`` are swapped for the CUDA modules.  Passed through as they are: postprocessors, custom embeddings
    and every other module (other output heads); a passed-through module that reads the number of systems from ``idx_m``
    keeps its host read."""
    in_mods = []
    for m in model.input_modules:
        n = type(m).__name__
        if n == "PairwiseDistances":
            in_mods.append(atomistic.PairwiseDistances())
        elif n == "FilterShortRange":
            in_mods.append(atomistic.FilterShortRange(float(m.short_range_cutoff)))
        else:
            in_mods.append(m)
    out_mods = []
    for m in model.output_modules:
        n = type(m).__name__
        if n == "Atomwise" and m.n_out == 1 and len(m.outnet) == 2:
            act = _map_act(m.outnet[0].activation)
            new = atomistic.Atomwise(m.outnet[0].in_features, 1, n_hidden=m.outnet[0].out_features, n_layers=2,
                                     activation=act, aggregation_mode=m.aggregation_mode, output_key=m.output_key,
                                     per_atom_output_key=m.per_atom_output_key)
            new.load_state_dict(m.state_dict())
            out_mods.append(new)
        elif n == "Forces":
            out_mods.append(atomistic.Forces(m.calc_forces, m.calc_stress, m.energy_key, m.force_key, m.stress_key))
        elif n in ("DipoleMoment", "Polarizability"):
            out_mods.append(_convert_head(m))
        elif n in ("ZBLRepulsionEnergy", "EnergyCoulomb"):
            out_mods.append(_convert_pair_term(m))
        elif n == "EnergyEwald":
            out_mods.append(_convert_ewald(m))
        elif n == "Aggregation":
            out_mods.append(atomistic.Aggregation(list(m.keys), m.output_key))
        else:
            out_mods.append(m)
    new = NeuralNetworkPotential(_convert_representation(model.representation), in_mods, out_mods,
                                 list(model.postprocessors), getattr(model, "input_dtype_str", "float32"),
                                 getattr(model, "do_postprocessing", True))
    was_double = any(p.dtype == torch.float64 for p in model.parameters())
    new.float()                  # the kernels compute in fp32 (weights copied through state_dict are cast on load)
    if was_double:
        new.cast_inputs = True
        new.input_dtype_str = "float32"
    new.eval()
    return new


# module lists of the representations that ``shared_interactions`` replicates (one module under every index)
SHARED_BLOCK_KEYS = r"\.(interactions|mixing|so3convs|mixings1|mixings2|mixings3|gatings)\.\d+\."


def from_spec(spec: dict, params: Optional[dict] = None, device=None) -> NeuralNetworkPotential:
    """Assemble [PairwiseDistances] -> {PaiNN|SchNet|SO3net} -> [Atomwise(energy), Forces] from a ``synthetic.model_spec``
    dictionary and (optionally) a flat weight dictionary with the reference ``state_dict`` keys."""
    import numpy as np

    if spec["rbf"] == "gaussian":
        rbf = snn.GaussianRBF(n_rbf=spec["n_rbf"], cutoff=spec["cutoff"])
    else:
        rbf = snn.BesselRBF(n_rbf=spec["n_rbf"], cutoff=spec["cutoff"])
    cut = snn.CosineCutoff(spec["cutoff"])
    if spec["kind"] == "painn":
        rep = representation.PaiNN(spec["n_atom_basis"], spec["n_interactions"], rbf, cut,
                                   shared_interactions=spec["shared_interactions"],
                                   shared_filters=spec["shared_filters"], epsilon=spec["epsilon"])
    elif spec["kind"] == "so3net":
        rep = representation.SO3net(spec["n_atom_basis"], spec["n_interactions"], spec["lmax"], rbf, cut,
                                    shared_interactions=spec["shared_interactions"],
                                    return_vector_representation=bool(spec.get("return_vector_representation", False)))
    else:
        rep = representation.SchNet(spec["n_atom_basis"], spec["n_interactions"], rbf, cut,
                                    n_filters=spec["n_filters"], shared_interactions=spec["shared_interactions"])
    outs: List[nn.Module] = [atomistic.Atomwise(n_in=spec["n_atom_basis"], output_key="energy")]
    want_stress = bool(spec.get("stress", False))
    if spec.get("forces", True) or want_stress:
        outs.append(atomistic.Forces(calc_forces=bool(spec.get("forces", True)), calc_stress=want_stress,
                                     energy_key="energy", force_key="forces"))
    ins: List[nn.Module] = ([atomistic.Strain()] if want_stress else []) + [atomistic.PairwiseDistances()]
    model = NeuralNetworkPotential(rep, ins, outs, postprocessors=[], do_postprocessing=False)
    if params is not None:
        import re
        sd = model.state_dict()
        new = {}
        for k in sd:
            kk = k
            if k not in params and spec["shared_interactions"]:
                kk = re.sub(SHARED_BLOCK_KEYS, r".\1.0.", k)
            new[k] = torch.as_tensor(np.asarray(params[kk])).to(sd[k].dtype)
        model.load_state_dict(new)
    model.eval()
    if device is not None:
        model = model.to(device)
    return model


def batch_to_device(batch: dict, device, pin: bool = False) -> Dict[str, torch.Tensor]:
    """numpy batch (``synthetic``) -> dict of tensors on ``device`` (fp32 / int64 like the reference's collate)."""
    out = {}
    for k, v in batch.items():
        t = torch.as_tensor(v)
        if t.is_floating_point():
            t = t.float()
        if pin:
            t = t.pin_memory()
        out[k] = t.to(device, non_blocking=pin)
    return out


class GraphedPotential:
    """CUDA-graph replay of a whole ``model(inputs)`` evaluation (energy, forces, graph-view build included) for a fixed
    problem shape -- SURVEY.md §8 f2.  The first call with a new shape signature (tensor shapes/dtypes of the batch) runs
    two eager warm-ups and captures the evaluation on a side stream into static buffers; later calls copy the batch into
    those buffers (``copy_``, asynchronous from pinned host memory), replay the graph and return the static outputs.

    Everything inside the model is capture-safe: the C-ABI calls only enqueue on the current stream, the receiver/sender
    views are rebuilt by captured kernels from the *current contents* of ``_idx_i/_idx_j`` on every replay, and no host
    synchronisation happens on the path (``_n_atoms`` supplies the number of systems).
    """

    def __init__(self, model: nn.Module, warmup: int = 2):
        self.model = model
        self.warmup = warmup
        self._cache = {}
        self._last = None

    @staticmethod
    def _signature(inputs: Dict[str, torch.Tensor]):
        return tuple(sorted((k, tuple(v.shape), str(v.dtype)) for k, v in inputs.items()))

    def _capture(self, inputs: Dict[str, torch.Tensor]):
        from . import ops

        dev = next(self.model.parameters()).device
        static_in = {k: v.detach().to(dev, copy=True) for k, v in inputs.items()}   # host (pinned) or device batches

        def run():
            ops._GRAPH_CACHE.clear()                 # the CSR/sender-view build must be part of the captured work
            # hand the model views of the static buffers: it marks positions as requiring grad, the buffers stay plain
            x = {k: (v.detach() if v.is_floating_point() else v) for k, v in static_in.items()}
            return self.model(x)

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = run()
        if isinstance(out, tuple):                   # NNEnsemble: (means, stds)
            static_out = tuple({k: v.detach() for k, v in o.items()} for o in out)
        else:
            static_out = {k: v.detach() for k, v in out.items()}
        return graph, static_in, static_out

    def __call__(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        sig = self._signature(inputs)
        entry = self._cache.get(sig)
        if entry is None:
            entry = self._capture(inputs)
            self._cache[sig] = entry
        graph, static_in, static_out = entry
        for k, v in inputs.items():
            static_in[k].copy_(v, non_blocking=True)
        graph.replay()
        if properties.virial in inputs:             # the caller's virial buffer is an output: hand the replay's back
            inputs[properties.virial].copy_(static_in[properties.virial], non_blocking=True)
        self._last = entry
        return static_out

    def replay(self) -> Dict[str, torch.Tensor]:
        """Re-evaluate the batch that already sits in the static device buffers of the last call (no input copies):
        the device-resident loop of an MD driver that updates ``_positions`` in place, or a benchmark."""
        graph, _, static_out = self._last
        graph.replay()
        return static_out

    def static_inputs(self) -> Dict[str, torch.Tensor]:
        """The static device buffers of the last call (write new positions / neighbour lists into them, then ``replay``)."""
        return self._last[1]
