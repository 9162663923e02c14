"""LayerNorm / RMSNorm modules backed by the sm_90a kernels in ``unicore.ops``.

Parity: reference ``unicore/modules/layer_norm.py:50-82`` and ``rms_norm.py:82-135`` (always
affine, eps 1e-5, fp32 statistics).  Unlike the reference there is no hidden-size whitelist: the
kernels handle any last-dimension size.
"""
import numbers

import torch
from torch import nn
from torch.nn import init

from unicore import ops


def _as_shape(normalized_shape):
    if isinstance(normalized_shape, numbers.Integral):
        normalized_shape = (normalized_shape,)
    return torch.Size(normalized_shape)


class LayerNorm(nn.Module):
    def __init__(self, normalized_shape, eps=1e-5, elementwise_affine=True):
        super().__init__()
        if not elementwise_affine:
            raise ValueError("LayerNorm is always affine in unicore")
        self.normalized_shape = _as_shape(normalized_shape)
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(*self.normalized_shape))
        self.bias = nn.Parameter(torch.zeros(*self.normalized_shape))

    def reset_parameters(self):
        init.ones_(self.weight)
        init.zeros_(self.bias)

    def forward(self, input):
        return ops.layer_norm(input, self.normalized_shape, self.weight, self.bias, self.eps)

    def extra_repr(self):
        return "{}, eps={}, elementwise_affine=True".format(tuple(self.normalized_shape), self.eps)


class RMSNorm(nn.Module):
    def __init__(self, normalized_shape, eps=1e-5, elementwise_affine=True):
        super().__init__()
        if not elementwise_affine:
            raise ValueError("RMSNorm is always affine in unicore")
        self.normalized_shape = _as_shape(normalized_shape)
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(*self.normalized_shape))

    def reset_parameters(self):
        init.ones_(self.weight)

    def forward(self, input):
        return ops.rms_norm(input, self.normalized_shape, self.weight, self.eps)

    def extra_repr(self):
        return "{}, eps={}, elementwise_affine=True".format(tuple(self.normalized_shape), self.eps)


class FusedLayerNormFastFunction:
    """Call-compatible stand-in for the reference autograd Function (``layer_norm.py:22-48``): user code that
    calls ``FusedLayerNormFastFunction.apply(x, w, b, shape, eps)`` lands on the same kernels as the module."""

    @staticmethod
    def apply(input, weight, bias, normalized_shape, eps):
        return ops.layer_norm(input, _as_shape(normalized_shape), weight, bias, eps)


class FusedRMSNormFastFunction:
    """``FusedRMSNormFastFunction.apply(x, w, shape, eps)`` (reference ``rms_norm.py:24-50``)."""

    @staticmethod
    def apply(input, weight, normalized_shape, eps):
        return ops.rms_norm(input, _as_shape(normalized_shape), weight, eps)
