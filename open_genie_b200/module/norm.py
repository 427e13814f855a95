"""Normalisation / activation modules — mirrors genie/module/norm.py and the nn.GroupNorm / nn.SiLU
entries of the blueprint registry (genie/module/__init__.py:56-68)."""
from __future__ import annotations

import torch
import torch.nn as nn
from torch import Tensor

from .. import ops


class GroupNorm(nn.GroupNorm):
    """Blueprint 'group_norm' (genie/tokenizer.py:75-78): nn.GroupNorm's parameters, fused CUDA kernels."""

    def forward(self, x: Tensor) -> Tensor:
        return ops.group_norm_act(x, self.weight, self.bias, self.num_groups, self.eps, 'none')


class SiLU(nn.Module):
    """Blueprint 'silu' (genie/tokenizer.py:79)."""

    def forward(self, x: Tensor) -> Tensor:
        return ops.silu(x)


class AdaptiveGroupNorm(nn.Module):
    """GN(x) * Linear(mean(cond)) + Linear(mean(cond)) — genie/module/norm.py:8-69.
    state_dict keys: weight, bias, std.{weight,bias}, avg.{weight,bias}; same init (norm.py:43-53).

    The conditioning path (mean over the latent grid, two (B, dim_cond) -> (B, C) projections) is one fused kernel each way
    (ops.adagn_condition); the modulation itself is folded into the same per-(sample, channel) scale/shift pass as the
    GroupNorm."""

    def __init__(self, dim_cond: int, num_groups: int, num_channels: int, cond_bias: bool = True, affine: bool = True,
                 eps: float = 1e-5, device=None, dtype=None) -> None:
        super().__init__()
        if num_channels % num_groups != 0:
            raise ValueError('num_channels must be divisible by num_groups')
        self.num_groups, self.num_channels, self.eps, self.affine = num_groups, num_channels, eps, affine
        kw = {'device': device, 'dtype': dtype}
        if affine:
            self.weight = nn.Parameter(torch.ones(num_channels, **kw))
            self.bias = nn.Parameter(torch.zeros(num_channels, **kw))
        else:
            self.register_parameter('weight', None)
            self.register_parameter('bias', None)
        self.std = nn.Linear(dim_cond, num_channels)
        self.avg = nn.Linear(dim_cond, num_channels) if cond_bias else None
        nn.init.ones_(self.std.bias)
        nn.init.zeros_(self.std.weight)
        if self.avg is not None:
            nn.init.zeros_(self.avg.bias)
            nn.init.zeros_(self.avg.weight)

    def forward(self, inp: Tensor, cond: Tensor) -> Tensor:
        # 'b d ... -> b d (...)' .mean(-1), then the two Linear(dim_cond, C)  (norm.py:62-66): one fused launch
        std, avg = ops.adagn_condition(cond, self.std.weight, self.std.bias,
                                       self.avg.weight if self.avg is not None else None,
                                       self.avg.bias if self.avg is not None else None)
        return ops.group_norm_act(inp, self.weight, self.bias, self.num_groups, self.eps, 'none', std, avg)
