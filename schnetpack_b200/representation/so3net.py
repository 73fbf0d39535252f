"""SO3net on the CUDA kernels -- drop-in for ``schnetpack.representation.SO3net``.

Constructor signature, attributes, tensor-dict protocol and ``state_dict`` keys follow the reference
(representation/so3net.py:15-155); the arithmetic is the kernel pipeline of ``schnetpack_b200.functional.so3net_forward``
(fused convolution with the filter evaluated in-kernel, no [E, n_cg, F] temporaries).
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
from ..nn import so3

__all__ = ["SO3net"]


class SO3net(nn.Module):
    """SO(3)-equivariant representation from spherical harmonics and Clebsch-Gordan tensor products.

    Outputs ``scalar_representation`` [N, F], ``multipole_representation`` [N, (lmax+1)^2, F] and, with
    ``return_vector_representation``, ``vector_representation`` [N, 3, F] (the l = 1 rows in x, y, z order).  The kernels
    cover lmax <= 3, F a multiple of 4 up to 256, Gaussian or Bessel basis with CosineCutoff; ``activation`` is stored
    but unused (the gates are sigmoids), as in the reference."""

    def __init__(self, n_atom_basis: int, n_interactions: int, lmax: int, radial_basis: nn.Module,
                 cutoff_fn: Optional[Callable] = None, shared_interactions: bool = False,
                 return_vector_representation: bool = False, activation: Optional[Callable] = F.silu,
                 nuclear_embedding: Optional[nn.Module] = None, electronic_embeddings: Optional[List] = None):
        super().__init__()
        self.n_atom_basis = n_atom_basis
        self.n_interactions = n_interactions
        self.lmax = lmax
        self.cutoff_fn = cutoff_fn
        self.cutoff = cutoff_fn.cutoff
        self.radial_basis = radial_basis
        self.return_vector_representation = return_vector_representation
        self.activation = activation

        if nuclear_embedding is None:
            nuclear_embedding = nn.Embedding(100, n_atom_basis)
        self.embedding = nuclear_embedding
        if electronic_embeddings is None:
            electronic_embeddings = []
        self.electronic_embeddings = nn.ModuleList(electronic_embeddings)

        self.sphharm = so3.RealSphericalHarmonics(lmax=lmax)
        self.so3convs = snn.replicate_module(
            lambda: so3.SO3Convolution(lmax, n_atom_basis, self.radial_basis.n_rbf), n_interactions, shared_interactions)
        self.mixings1 = snn.replicate_module(lambda: nn.Linear(n_atom_basis, n_atom_basis, bias=False), n_interactions,
                                             shared_interactions)
        self.mixings2 = snn.replicate_module(lambda: nn.Linear(n_atom_basis, n_atom_basis, bias=False), n_interactions,
                                             shared_interactions)
        self.mixings3 = snn.replicate_module(lambda: nn.Linear(n_atom_basis, n_atom_basis, bias=False), n_interactions,
                                             shared_interactions)
        self.gatings = snn.replicate_module(lambda: so3.SO3ParametricGatedNonlinearity(n_atom_basis, lmax),
                                            n_interactions, shared_interactions)
        self.so3product = so3.SO3TensorProduct(lmax)
        self._pk = K.SO3netPack()

    # ---- kernel-side views of the configuration ------------------------------------------------------------------
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

    def _pack(self) -> K.SO3netPack:
        params = [p for p in self.parameters()]
        if self._pk.stale(params):
            self._pk.build(self)
            self._pk.mark(params)
        return self._pk

    def _apply(self, fn, *a, **k):  # .to()/.cuda()/.float(): drop the cached kernel-side weights
        self._pk = K.SO3netPack()
        return super()._apply(fn, *a, **k)

    def _check_kernel_shapes(self):
        if self.lmax > so3.KERNEL_LMAX or self.lmax < 0:
            raise NotImplementedError(f"SO3net kernels support lmax <= {so3.KERNEL_LMAX} (got {self.lmax}); "
                                      "train() mode evaluates any lmax with ATen operations")
        if self.n_atom_basis % 4 or self.n_atom_basis > 256:
            raise NotImplementedError(f"SO3net kernels support n_atom_basis a multiple of 4 up to 256 "
                                      f"(got {self.n_atom_basis})")
        if not isinstance(self.radial_basis, (snn.GaussianRBF, snn.BesselRBF)) or not isinstance(
                self.cutoff_fn, snn.CosineCutoff):
            raise NotImplementedError("SO3net kernels support GaussianRBF/BesselRBF x CosineCutoff")

    @ops.on_tensor_device
    def forward(self, inputs: Dict[str, torch.Tensor]):
        atomic_numbers = inputs[properties.Z]
        r_ij = inputs[properties.Rij]
        idx_i = inputs[properties.idx_i]
        idx_j = inputs[properties.idx_j]
        n_atoms = atomic_numbers.shape[0]
        if snn.use_training_path(self):
            from .. import functional_torch as T

            return T.so3net(self, inputs)
        self._check_kernel_shapes()
        graph = ops.get_graph(idx_i, idx_j, n_atoms)

        if isinstance(self.embedding, nn.Embedding) and len(self.electronic_embeddings) == 0:
            x0 = ops.embedding(self.embedding.weight.detach().contiguous(), atomic_numbers)     # so3net.py:130
        else:  # user-supplied embedding modules run as given (so3net.py:130-132)
            x0 = self.embedding(atomic_numbers)
            for embedding in self.electronic_embeddings:
                x0 = x0 + embedding(x0, inputs)
            x0 = x0.detach().contiguous()

        holder = dict(module=self, graph=graph)
        q, x = K.SO3netFunction.apply(r_ij if r_ij.is_contiguous() else r_ij.contiguous(), x0, holder)
        inputs["scalar_representation"] = q
        inputs["multipole_representation"] = x
        if self.return_vector_representation:                   # l = 1 rows [y, z, x] -> [x, y, z]
            inputs["vector_representation"] = torch.roll(x[:, 1:4], 1, 1)
        return inputs
