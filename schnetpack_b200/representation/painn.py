"""PaiNN representation on the CUDA kernels -- drop-in for ``schnetpack.representation.PaiNN``.

Constructor signature, attributes, tensor-dict protocol and ``state_dict`` keys follow
/root/reference/src/schnetpack/representation/painn.py:120-256; the arithmetic is the fused kernel pipeline of
``schnetpack_b200.functional.painn_forward`` (no ``[E,3F]`` temporaries, filter recomputed per edge in-kernel).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import functional as K
from .. import nn as snn
from .. import ops
from .. import properties

__all__ = ["PaiNN", "PaiNNInteraction", "PaiNNMixing"]


class PaiNNInteraction(nn.Module):
    """One interaction block (painn.py:14-67): interatomic_context_net = Dense(F,F,act) -> Dense(F,3F).  Inside
    ``PaiNN.forward`` the block runs in the fused edge kernel (filter evaluated in-kernel); called directly with a
    materialised filter, as the reference's block API allows, it runs on ``spk_painn_edge_wij_{fwd,bwd}``."""

    def __init__(self, n_atom_basis: int, activation: Callable):
        super().__init__()
        self.n_atom_basis = n_atom_basis
        self.interatomic_context_net = nn.Sequential(
            snn.Dense(n_atom_basis, n_atom_basis, activation=activation),
            snn.Dense(n_atom_basis, 3 * n_atom_basis, activation=None),
        )

    @ops.on_tensor_device
    def forward(self, q, mu, Wij, dir_ij, idx_i, idx_j, n_atoms: int):
        """painn.py:31-67.  q [N,1,F], mu [N,3,F], Wij [E,1,3F], dir_ij [E,3] -> (q, mu); differentiable w.r.t. q, mu, Wij
        and dir_ij (first order)."""
        F_ = self.n_atom_basis
        x = self.interatomic_context_net(q)                                        # :54 (Dense kernels)
        graph = ops.get_graph(idx_i, idx_j, int(n_atoms))
        q1, mu1 = K.PaiNNEdgeWijFunction.apply(x.reshape(-1, 3 * F_), mu, q.reshape(-1, F_), Wij.reshape(-1, 3 * F_),
                                               dir_ij, graph, F_)                 # :55-65
        return q1.view(q.shape), mu1


class PaiNNMixing(nn.Module):
    """One mixing block (painn.py:70-117); callable on its own like the reference's."""

    def __init__(self, n_atom_basis: int, activation: Callable, epsilon: float = 1e-8):
        super().__init__()
        self.n_atom_basis = n_atom_basis
        self.intraatomic_context_net = nn.Sequential(
            snn.Dense(2 * n_atom_basis, n_atom_basis, activation=activation),
            snn.Dense(n_atom_basis, 3 * n_atom_basis, activation=None),
        )
        self.mu_channel_mix = snn.Dense(n_atom_basis, 2 * n_atom_basis, activation=None, bias=False)
        self.epsilon = epsilon
        self.activation = activation
        self._blk, self._sig = None, None

    def _apply(self, fn, *a, **k):
        self._blk, self._sig = None, None
        return super()._apply(fn, *a, **k)

    def _pack(self):
        params = list(self.parameters())
        sig = K.ParamPack.signature(params)
        if self._sig != sig:
            m0, m1 = self.intraatomic_context_net[0], self.intraatomic_context_net[1]
            self._blk = dict(mix=ops.Lin(self.mu_channel_mix.weight), m0=ops.Lin(m0.weight, m0.bias),
                             m1=ops.Lin(m1.weight, m1.bias))
            self._sig = sig
        return self._blk

    @ops.on_tensor_device
    def forward(self, q, mu):
        """painn.py:92-117.  q [N,1,F], mu [N,3,F] -> (q, mu)."""
        F_ = self.n_atom_basis
        if snn.use_training_path(self):
            raise NotImplementedError("PaiNNMixing called on its own in training mode: train through PaiNN.forward "
                                      "(functional_torch) or call .eval()")
        q2, mu2 = K.PaiNNMixingFunction.apply(q.reshape(-1, F_), mu, self._pack(), F_, float(self.epsilon),
                                              snn.activation_code(self.activation))
        return q2.view(q.shape), mu2


class PaiNN(nn.Module):
    """PaiNN - polarizable interaction neural network (painn.py:120-256), CUDA kernel path."""

    def __init__(self, n_atom_basis: int, n_interactions: int, radial_basis: nn.Module,
                 cutoff_fn: Optional[Callable] = None, activation: Optional[Callable] = F.silu,
                 shared_interactions: bool = False, shared_filters: bool = False, epsilon: float = 1e-8,
                 nuclear_embedding: Optional[nn.Module] = None, electronic_embeddings: Optional[List] = None):
        super().__init__()
        self.n_atom_basis = n_atom_basis
        self.n_interactions = n_interactions
        self.cutoff_fn = cutoff_fn
        self.cutoff = cutoff_fn.cutoff
        self.radial_basis = radial_basis
        self.activation = activation

        if nuclear_embedding is None:
            nuclear_embedding = nn.Embedding(100, n_atom_basis)
        self.embedding = nuclear_embedding
        if electronic_embeddings is None:
            electronic_embeddings = []
        self.electronic_embeddings = nn.ModuleList(electronic_embeddings)

        self.share_filters = shared_filters
        if shared_filters:
            self.filter_net = snn.Dense(self.radial_basis.n_rbf, 3 * n_atom_basis, activation=None)
        else:
            self.filter_net = snn.Dense(self.radial_basis.n_rbf, self.n_interactions * n_atom_basis * 3,
                                        activation=None)
        self.interactions = snn.replicate_module(
            lambda: PaiNNInteraction(n_atom_basis=self.n_atom_basis, activation=activation),
            self.n_interactions, shared_interactions)
        self.mixing = snn.replicate_module(
            lambda: PaiNNMixing(n_atom_basis=self.n_atom_basis, activation=activation, epsilon=epsilon),
            self.n_interactions, shared_interactions)
        self._pk = K.PaiNNPack()

    # ---- kernel-side views of the configuration ------------------------------------------------------------------
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

    def _pack(self) -> K.PaiNNPack:
        params = [p for p in self.parameters()]
        if self._pk.stale(params):
            self._pk.build(self)
            self._pk.mark(params)
        return self._pk

    def _apply(self, fn, *a, **k):  # .to()/.cuda()/.float(): drop the cached kernel-side weights
        self._pk = K.PaiNNPack()
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

            return T.painn(self, inputs)
        if not isinstance(self.radial_basis, (snn.GaussianRBF, snn.BesselRBF)) or not isinstance(
                self.cutoff_fn, snn.CosineCutoff):
            raise NotImplementedError("fused PaiNN kernels support GaussianRBF/BesselRBF x CosineCutoff")
        ops.check_painn_shape(self.n_atom_basis, self.radial_basis.n_rbf)
        graph = ops.get_graph(idx_i, idx_j, n_atoms)

        if isinstance(self.embedding, nn.Embedding) and len(self.electronic_embeddings) == 0:
            q0 = ops.embedding(self.embedding.weight.detach().contiguous(), atomic_numbers)   # painn.py:239
        else:  # user-supplied embedding modules run as given (painn.py:239-241)
            q0 = self.embedding(atomic_numbers)
            for embedding in self.electronic_embeddings:
                q0 = q0 + embedding(q0, inputs)
            q0 = q0.detach().contiguous()

        holder = dict(module=self, graph=graph)
        q, mu = K.PaiNNFunction.apply(r_ij if r_ij.is_contiguous() else r_ij.contiguous(), q0, holder)
        inputs["scalar_representation"] = q
        inputs["vector_representation"] = mu
        return inputs
