"""nn.Linear-compatible parameter holder whose forward runs on the wgmma GEMM kernel."""
from __future__ import annotations

import math

import torch
import torch.nn as nn
from torch import Tensor

from .. import ops
from .video import CONV_REGISTRY


class LinearRows(nn.Module):
    """y = x W^T + b over the last dim (keys 'weight' [N][K], 'bias'), K % 64 == 0. The bf16 operand copy is kept
    fresh by FusedAdamW (same registry as the conv layers) or re-cast when the parameter's version changes."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True) -> None:
        super().__init__()
        w = torch.empty(out_features, in_features)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        self.weight = nn.Parameter(w)
        if bias:
            bound = 1 / math.sqrt(in_features)
            self.bias = nn.Parameter(torch.empty(out_features).uniform_(-bound, bound))
        else:
            self.register_parameter('bias', None)
        self.in_features, self.out_features = in_features, out_features
        self._packed = None
        self._packed_key = None
        self._fused_into = None
        CONV_REGISTRY[id(self.weight)] = self

    def packed(self) -> Tensor:
        w = self.weight
        key = (w.data_ptr(), w._version, w.device)
        if self._packed is None or self._packed_key != key:
            if self._packed is None or self._packed.device != w.device:
                self._packed = torch.empty(w.shape, dtype=torch.bfloat16, device=w.device)
            ops._lib.call('og_copy_rows_to_bf16', w.data_ptr(), 1, w.shape[1], self._packed.data_ptr(), w.shape[1],
                          w.shape[0], w.shape[1], ops._stream())
            self._packed_key = key
        return self._packed

    def bf16_target(self):
        return self.packed(), 0

    def forward(self, x: Tensor, out_f32: bool = False) -> Tensor:
        ops._require_cuda(x, 'linear input')
        lead = x.shape[:-1]
        y = ops.linear_rows(x.reshape(-1, x.shape[-1]), self.weight, self.bias, self.packed(), out_f32)
        return y.reshape(*lead, self.out_features)
