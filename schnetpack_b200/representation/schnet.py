"""SchNet representation on the CUDA kernels -- drop-in for ``schnetpack.representation.SchNet``
(/root/reference/src/schnetpack/representation/schnet.py:73-173)."""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Union

import torch
from torch import nn

from .. import functional as K
from .. import nn as snn
from .. import ops
from .. import properties
from ..nn import Dense, shifted_softplus

__all__ = ["SchNet", "SchNetInteraction"]


class SchNetInteraction(nn.Module):
    """One interaction block (schnet.py:14-70): in2f (no bias), f2out = Dense(act) -> Dense, filter_network =
    Dense(n_rbf -> n_filters, act) -> Dense(n_filters -> n_filters).  ``SchNet.forward`` runs the block inside its own
    kernel pipeline; called directly (the reference's block API) it runs Dense kernels + ``spk_cfconv_{fwd,bwd}``."""

    def __init__(self, n_atom_basis: int, n_rbf: int, n_filters: int, activation: Callable = shifted_softplus):
        super().__init__()
        self.in2f = Dense(n_atom_basis, n_filters, bias=False, activation=None)
        self.f2out = nn.Sequential(
            Dense(n_filters, n_atom_basis, activation=activation),
            Dense(n_atom_basis, n_atom_basis, activation=None),
        )
        self.filter_network = nn.Sequential(
            Dense(n_rbf, n_filters, activation=activation), Dense(n_filters, n_filters)
        )

    @ops.on_tensor_device
    def forward(self, x, f_ij, idx_i, idx_j, rcut_ij):
        """schnet.py:41-70.  x [N,F], f_ij [E,n_rbf], rcut_ij [E] -> v [N,F]; differentiable w.r.t. x, f_ij, rcut_ij."""
        h = self.in2f(x)                                                           # :60
        Wij = self.filter_network(f_ij)                                            # :61
        graph = ops.get_graph(idx_i, idx_j, int(x.shape[0]))
        m = K.CFConvFunction.apply(h, Wij, rcut_ij, graph)                         # :62-67
        return self.f2out(m)                                                       # :69


class SchNet(nn.Module):
    """SchNet (schnet.py:73-173), CUDA kernel path."""

    def __init__(self, n_atom_basis: int, n_interactions: int, radial_basis: nn.Module, cutoff_fn: Callable,
                 n_filters: int = None, shared_interactions: bool = False,
                 activation: Union[Callable, nn.Module] = shifted_softplus,
                 nuclear_embedding: Optional[nn.Module] = None, electronic_embeddings: Optional[List] = None):
        super().__init__()
        self.n_atom_basis = n_atom_basis
        self.n_filters = n_filters or self.n_atom_basis
        self.radial_basis = radial_basis
        self.cutoff_fn = cutoff_fn
        self.cutoff = cutoff_fn.cutoff
        self.activation = activation

        if nuclear_embedding is None:
            nuclear_embedding = nn.Embedding(100, n_atom_basis)
        self.embedding = nuclear_embedding
        if electronic_embeddings is None:
            electronic_embeddings = []
        self.electronic_embeddings = nn.ModuleList(electronic_embeddings)

        self.interactions = snn.replicate_module(
            lambda: SchNetInteraction(n_atom_basis=self.n_atom_basis, n_rbf=self.radial_basis.n_rbf,
                                      n_filters=self.n_filters, activation=activation),
            n_interactions, shared_interactions)
        self._pk = K.SchNetPack()

    @property
    def _act(self):
        return snn.activation_code(self.activation)

    @property
    def _n_rbf(self):
        return self.radial_basis.n_rbf

    @property
    def _rbf_kind(self):
        return self.radial_basis.kind

    @property
    def _rbf_p0(self):
        return self.radial_basis.kernel_params()[0]

    @property
    def _rbf_p1(self):
        return self.radial_basis.kernel_params()[1]

    @property
    def _cutoff_value(self):
        return self.cutoff_fn.value()

    def _pack(self) -> K.SchNetPack:
        params = [p for p in self.parameters()]
        if self._pk.stale(params):
            self._pk.build(self)
            self._pk.mark(params)
        return self._pk

    def _apply(self, fn, *a, **k):
        self._pk = K.SchNetPack()
        return super()._apply(fn, *a, **k)

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]):
        atomic_numbers = inputs[properties.Z]
        r_ij = inputs[properties.Rij]
        idx_i = inputs[properties.idx_i]
        idx_j = inputs[properties.idx_j]
        n_atoms = atomic_numbers.shape[0]
        if snn.use_training_path(self):           # training (weight gradients, double backward): ATen path, SURVEY 8 f3
            from .. import functional_torch as T

            return T.schnet(self, inputs)
        if not isinstance(self.radial_basis, (snn.GaussianRBF, snn.BesselRBF)) or not isinstance(
                self.cutoff_fn, snn.CosineCutoff):
            raise NotImplementedError("fused SchNet kernels support GaussianRBF/BesselRBF x CosineCutoff")
        need_grad = r_ij.requires_grad and torch.is_grad_enabled()
        ops.check_schnet_shape(self.n_filters, self.radial_basis.n_rbf, need_grad)
        # inference on the fused forward kernels builds its own receiver view over the ACTIVE edges (d < cutoff) from r_ij
        fused = (not need_grad
                 and ops.cfconv_tc_ok(self.n_atom_basis, self.n_filters, self.radial_basis.n_rbf, r_ij.shape[0]))
        graph = None if fused else ops.get_graph(idx_i, idx_j, n_atoms)
        if isinstance(self.embedding, nn.Embedding) and len(self.electronic_embeddings) == 0:
            x0 = ops.embedding(self.embedding.weight.detach().contiguous(), atomic_numbers)   # schnet.py:161
        else:
            x0 = self.embedding(atomic_numbers)
            for embedding in self.electronic_embeddings:
                x0 = x0 + embedding(x0, inputs)
            x0 = x0.detach().contiguous()
        x = K.SchNetFunction.apply(r_ij if r_ij.is_contiguous() else r_ij.contiguous(), x0,
                                   dict(module=self, graph=graph, idx_i=idx_i, idx_j=idx_j))
        inputs["scalar_representation"] = x
        return inputs
