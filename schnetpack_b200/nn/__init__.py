"""Mirror of the reference's ``schnetpack.nn`` primitives that sit on the hot path, backed by the sm_90a CUDA kernels.

Same constructor signatures, buffers/parameters and ``state_dict`` keys as
/root/reference/src/schnetpack/nn/{radial,cutoff,base,activations,scatter,blocks,utils}.py.  Forward passes on CUDA
tensors launch the kernels of ``csrc/geometry.cu`` / ``csrc/gemm.cu``; first-order input gradients are provided
(that is what forces need); weight gradients are not (training = SURVEY.md §8 f3).
"""
from __future__ import annotations

import math
from typing import Callable, Optional, Sequence, Union

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.init import xavier_uniform_, zeros_

from .. import ops

__all__ = ["GaussianRBF", "BesselRBF", "CosineCutoff", "cosine_cutoff", "gaussian_rbf", "Dense", "shifted_softplus",
           "scatter_add", "build_mlp", "replicate_module", "activation_code", "use_training_path", "GatedEquivariantBlock",
           "build_gated_equivariant_mlp", "SwitchFunction"]


def use_training_path(module: nn.Module) -> bool:
    """True when ``module`` must take the differentiable ATen path of ``functional_torch`` instead of the kernels: it is in
    ``train()`` mode, grad mode is on and it has trainable parameters.  The CUDA path provides first-order input gradients
    (forces, stress) only; weight gradients and the double backward of force training (``create_graph``, SURVEY.md section 8
    f3) come from that path -- never silently from the kernels."""
    return module.training and torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters())


# ------------------------------------------------------------------------------------------------- activations
class _ActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, code):
        y, dy = ops.activation(x.detach().contiguous(), code, need_grad=x.requires_grad)
        ctx.dy = dy
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        return g * ctx.dy, None


def shifted_softplus(x: torch.Tensor):
    """nn/activations.py:9-22: softplus(x) - ln 2."""
    if x.is_cuda and x.dtype == torch.float32:
        return _ActFn.apply(x, ops.ACT_SSP)
    raise RuntimeError("schnetpack_b200.nn.shifted_softplus: fp32 CUDA tensors only (no CPU fallback)")


def activation_code(act) -> int:
    """Map an activation callable of the reference API onto a kernel epilogue code."""
    if act is None or isinstance(act, nn.Identity):
        return ops.ACT_NONE
    if act is F.silu or isinstance(act, nn.SiLU):
        return ops.ACT_SILU
    name = getattr(act, "__name__", type(act).__name__)
    if act is shifted_softplus or name == "shifted_softplus":
        return ops.ACT_SSP
    if name == "silu":
        return ops.ACT_SILU
    raise NotImplementedError(f"activation {act!r} has no fused kernel epilogue (supported: silu, shifted_softplus)")


# ------------------------------------------------------------------------------------------------- radial / cutoff
class _RbfFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, d, kind, p0, p1):
        out, dout = ops.rbf(d.detach().contiguous(), kind, p0, p1, need_grad=d.requires_grad)
        ctx.dout = dout
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        return (g * ctx.dout).sum(-1), None, None, None


def gaussian_rbf(inputs: torch.Tensor, offsets: torch.Tensor, widths: torch.Tensor):
    """nn/radial.py:11-15."""
    return _RbfFn.apply(inputs, ops.RBF_GAUSSIAN, offsets.detach().contiguous(), widths.detach().contiguous())


class GaussianRBF(nn.Module):
    """nn/radial.py:18-48 -- Gaussian radial basis, offsets = linspace(start, cutoff, n_rbf), shared width."""

    def __init__(self, n_rbf: int, cutoff: float, start: float = 0.0, trainable: bool = False):
        super().__init__()
        self.n_rbf = n_rbf
        offset = torch.linspace(start, cutoff, n_rbf)
        widths = torch.FloatTensor(torch.abs(offset[1] - offset[0]) * torch.ones_like(offset))
        if trainable:
            self.widths = nn.Parameter(widths)
            self.offsets = nn.Parameter(offset)
        else:
            self.register_buffer("widths", widths)
            self.register_buffer("offsets", offset)

    kind = ops.RBF_GAUSSIAN

    def kernel_params(self):
        return self.offsets.detach().contiguous(), self.widths.detach().contiguous()

    def forward(self, inputs: torch.Tensor):
        return gaussian_rbf(inputs, self.offsets, self.widths)


class BesselRBF(nn.Module):
    """nn/radial.py:82-110 -- sin(k pi d / rc) / d."""

    def __init__(self, n_rbf: int, cutoff: float):
        super().__init__()
        self.n_rbf = n_rbf
        freqs = torch.arange(1, n_rbf + 1) * math.pi / cutoff
        self.register_buffer("freqs", freqs)

    kind = ops.RBF_BESSEL

    def kernel_params(self):
        return self.freqs.detach().float().contiguous(), None

    def forward(self, inputs: torch.Tensor):
        return _RbfFn.apply(inputs, ops.RBF_BESSEL, self.freqs.detach().float().contiguous(), None)


class _CutoffFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, d, rc):
        out, dout = ops.cosine_cutoff(d.detach().contiguous(), rc, need_grad=d.requires_grad)
        ctx.dout = dout
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        return g * ctx.dout, None


def cosine_cutoff(input: torch.Tensor, cutoff: torch.Tensor):
    """nn/cutoff.py:14-33."""
    return _CutoffFn.apply(input, float(cutoff))


class CosineCutoff(nn.Module):
    """nn/cutoff.py:36-57 -- Behler cosine cutoff, buffer ``cutoff`` of shape [1]."""

    def __init__(self, cutoff: float):
        super().__init__()
        self.register_buffer("cutoff", torch.FloatTensor([cutoff]))
        self._v, self._vkey = float(cutoff), None

    def value(self) -> float:
        """Python float of the ``cutoff`` buffer (one host read per change of the buffer, e.g. after loading)."""
        key = (self.cutoff.data_ptr(), self.cutoff._version)
        if self._vkey != key:
            self._v = float(self.cutoff)
            self._vkey = key
        return self._v

    def forward(self, input: torch.Tensor):
        return _CutoffFn.apply(input, self.value())


def _switch_component(x: torch.Tensor, ones: torch.Tensor, zeros: torch.Tensor) -> torch.Tensor:
    """nn/cutoff.py:107-122."""
    x_ = torch.where(x <= 0, ones, x)
    return torch.where(x <= 0, zeros, torch.exp(-ones / x_))


class SwitchFunction(nn.Module):
    """nn/cutoff.py:125-158 -- decays from 1 to 0 between ``switch_on`` and ``switch_off`` (buffers of shape [1]).  Plain
    tensor algebra: the Coulomb kernels of csrc/pair_energy.cu evaluate it in-kernel from the two buffers."""

    def __init__(self, switch_on: float, switch_off: float):
        super().__init__()
        self.register_buffer("switch_on", torch.Tensor([switch_on]))
        self.register_buffer("switch_off", torch.Tensor([switch_off]))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = (x - self.switch_on) / (self.switch_off - self.switch_on)
        ones = torch.ones_like(x)
        zeros = torch.zeros_like(x)
        fp = _switch_component(x, ones, zeros)
        fm = _switch_component(1 - x, ones, zeros)
        return torch.where(x <= 0, ones, torch.where(x >= 1, zeros, fm / (fp + fm)))


# ------------------------------------------------------------------------------------------------- dense / mlp
class _DenseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, code):
        shp = x.shape
        x2 = x.detach().reshape(-1, shp[-1]).contiguous()
        need = x.requires_grad
        ctx.pre = None
        with ops.device_of(x2, weight):
            lin = ops.Lin(weight, bias)
            if need:
                y, ctx.pre = lin.fwd(x2, code, save_deriv=True)
            else:
                y = lin.fwd(x2, code)
        ctx.lin = lin
        ctx.code = code
        ctx.shp = shp
        return y.view(*shp[:-1], weight.shape[0])

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        g2 = g.reshape(-1, g.shape[-1]).contiguous()
        with ops.device_of(g2):
            gx = ctx.lin.bwd(g2, a_pre=ctx.pre if ctx.code != ops.ACT_NONE else None, a_act=ops.ACT_GIVEN)
        return gx.view(*ctx.shp), None, None, None


class Dense(nn.Linear):
    """nn/base.py:14-55 -- y = activation(x W^T + b); xavier-uniform weight, zero bias."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True,
                 activation: Union[Callable, nn.Module] = None, weight_init: Callable = xavier_uniform_,
                 bias_init: Callable = zeros_):
        self.weight_init = weight_init
        self.bias_init = bias_init
        super().__init__(in_features, out_features, bias)
        self.activation = activation
        if self.activation is None:
            self.activation = nn.Identity()

    def reset_parameters(self):
        self.weight_init(self.weight)
        if self.bias is not None:
            self.bias_init(self.bias)

    def forward(self, input: torch.Tensor):
        if use_training_path(self):               # training: differentiable ATen path (functional_torch)
            from .. import functional_torch as T

            return T.dense(input, self, T._activation(self.activation))
        return _DenseFn.apply(input, self.weight, self.bias, activation_code(self.activation))


def build_mlp(n_in: int, n_out: int, n_hidden: Optional[Union[int, Sequence[int]]] = None, n_layers: int = 2,
              activation: Callable = F.silu, last_bias: bool = True, last_zero_init: bool = False) -> nn.Module:
    """nn/blocks.py:12-76 -- pyramidal (n_hidden None) or rectangular MLP of Dense layers."""
    if n_hidden is None:
        c_neurons = n_in
        n_neurons = []
        for _ in range(n_layers):
            n_neurons.append(c_neurons)
            c_neurons = max(n_out, c_neurons // 2)
        n_neurons.append(n_out)
    else:
        if type(n_hidden) is int:
            n_hidden = [n_hidden] * (n_layers - 1)
        else:
            n_hidden = list(n_hidden)
        n_neurons = [n_in] + n_hidden + [n_out]
    layers = [Dense(n_neurons[i], n_neurons[i + 1], activation=activation) for i in range(n_layers - 1)]
    if last_zero_init:
        layers.append(Dense(n_neurons[-2], n_neurons[-1], activation=None, weight_init=torch.nn.init.zeros_,
                            bias=last_bias))
    else:
        layers.append(Dense(n_neurons[-2], n_neurons[-1], activation=None, bias=last_bias))
    return nn.Sequential(*layers)


class GatedEquivariantBlock(nn.Module):
    """nn/equivariant.py:11-71 -- gated mixing of scalar [N, n_sin] and vector [N, 3, n_vin] features.  Called on its own
    it evaluates the ATen formula on any device; inside ``atomistic.DipoleMoment`` / ``Polarizability`` in ``eval()`` mode
    its weights run on the kernels of ``csrc/equivariant.cu``."""

    def __init__(self, n_sin: int, n_vin: int, n_sout: int, n_vout: int, n_hidden: int, activation=F.silu,
                 sactivation=None):
        super().__init__()
        self.n_sin = n_sin
        self.n_vin = n_vin
        self.n_sout = n_sout
        self.n_vout = n_vout
        self.n_hidden = n_hidden
        self.mix_vectors = Dense(n_vin, 2 * n_vout, activation=None, bias=False)
        self.scalar_net = nn.Sequential(Dense(n_sin + n_vout, n_hidden, activation=activation),
                                        Dense(n_hidden, n_sout + n_vout, activation=None))
        self.sactivation = sactivation

    def forward(self, inputs):
        from .. import functional_torch as T

        return T.gated_block(self, *inputs)


def build_gated_equivariant_mlp(n_in: int, n_out: int, n_hidden: Optional[Union[int, Sequence[int]]] = None,
                                n_gating_hidden: Optional[Union[int, Sequence[int]]] = None, n_layers: int = 2,
                                activation: Callable = F.silu, sactivation: Callable = F.silu) -> nn.Module:
    """nn/blocks.py:79-156 -- MLP of GatedEquivariantBlocks; the last block has no scalar activation."""
    if n_hidden is None:
        c_neurons = n_in
        n_neurons = []
        for _ in range(n_layers):
            n_neurons.append(c_neurons)
            c_neurons = max(n_out, c_neurons // 2)
        n_neurons.append(n_out)
    else:
        if type(n_hidden) is int:
            n_hidden = [n_hidden] * (n_layers - 1)
        else:
            n_hidden = list(n_hidden)
        n_neurons = [n_in] + n_hidden + [n_out]
    if n_gating_hidden is None:
        n_gating_hidden = n_neurons[:-1]
    elif type(n_gating_hidden) is int:
        n_gating_hidden = [n_gating_hidden] * n_layers
    else:
        n_gating_hidden = list(n_gating_hidden)
    layers = [GatedEquivariantBlock(n_neurons[i], n_neurons[i], n_neurons[i + 1], n_neurons[i + 1], n_gating_hidden[i],
                                    activation=activation, sactivation=sactivation) for i in range(n_layers - 1)]
    layers.append(GatedEquivariantBlock(n_neurons[-2], n_neurons[-2], n_neurons[-1], n_neurons[-1], n_gating_hidden[-1],
                                        activation=activation, sactivation=None))
    return nn.Sequential(*layers)


def replicate_module(module_factory: Callable[[], nn.Module], n: int, share_params: bool):
    """nn/utils.py:11-18."""
    if share_params:
        return nn.ModuleList([module_factory()] * n)
    return nn.ModuleList([module_factory() for _ in range(n)])


# ------------------------------------------------------------------------------------------------- scatter_add
class _ScatterAddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, idx, dim_size):
        # group rows by idx on device (same builder as the edge graph: idx plays the receiver role)
        g = ops.EdgeGraph(idx, idx, dim_size)
        ctx.idx = idx
        return ops.segment_sum(x.detach().contiguous(), g.rowptr, g.slot_eid, dim_size)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        return g.index_select(0, ctx.idx), None, None


def scatter_add(x: torch.Tensor, idx_i: torch.Tensor, dim_size: int, dim: int = 0) -> torch.Tensor:
    """nn/scatter.py:7-34 -- deterministic segmented sum (the reference's index_add uses fp32 atomics on GPU)."""
    if dim != 0:
        return _ScatterAddFn.apply(x.transpose(0, dim).contiguous(), idx_i, dim_size).transpose(0, dim)
    return _ScatterAddFn.apply(x, idx_i, dim_size)
