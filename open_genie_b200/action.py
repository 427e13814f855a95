"""LatentAction — mirrors genie/action.py:31-176 (same constructor, encode/decode/forward/sample, return tuples,
state_dict keys) on the CUDA kernels.

Pinned to the HEAD-valid behaviour (SURVEY.md §8): the reference constructor forgets `input_dim` when it builds
the quantizer (action.py:93-101), which makes LookupFreeQuantization project from 2^d inputs and crash in
forward; here the quantizer is built with input_dim = d_codebook, i.e. proj_inp / proj_out are Identity —
exactly what the pinned reference run patches in.
"""
from __future__ import annotations

from math import prod
from typing import Tuple

import torch
import torch.nn as nn
from torch import Tensor

from . import ops
from .module import parse_blueprint
from .module.linear import LinearRows
from .module.quantization import LookupFreeQuantization
from .module.video import CausalConv3d, Downsample, Upsample
from .utils import Blueprint


class _ToActLinear(nn.Module):
    """nn.Linear(K, d, bias=False) of `to_act` (action.py:83-90) applied to 'b c t ... -> b t (c ...)'.
    The activations are NDHWC, so per frame they flatten as (h, w, c); the weight keeps the reference's (c, h, w)
    column order in the state_dict and is permuted when the bf16 operand is cast (a few MB per step)."""

    def __init__(self, in_features: int, out_features: int) -> None:
        super().__init__()
        lin = nn.Linear(in_features, out_features, bias=False)
        self.weight = nn.Parameter(lin.weight.detach().clone())
        self.in_features, self.out_features = in_features, out_features

    def forward(self, video: Tensor) -> Tensor:
        # video: internal (B, C, T, h, w)  ->  act logits (B, T, d) fp32
        B, C, T, h, w = video.shape
        x = video.permute(0, 2, 3, 4, 1)                         # (B, T, h, w, C) contiguous view
        if x.dtype != torch.bfloat16 or not x.is_contiguous():
            x = x.to(torch.bfloat16).contiguous()
        n = self.out_features
        w_perm = self.weight.view(n, C, h, w).permute(0, 2, 3, 1).reshape(n, h * w * C)    # (h, w, c) column order
        packed = w_perm.detach().to(torch.bfloat16).contiguous()
        y = ops.linear_rows(x.reshape(B * T, h * w * C), w_perm.contiguous(), None, packed, out_f32=True)
        return y.reshape(B, T, n)


class LatentAction(nn.Module):
    def __init__(self, enc_desc: Blueprint, dec_desc: Blueprint, d_codebook: int, inp_channels: int = 3,
                 inp_shape=(64, 64), ker_size=3, n_embd: int = 256, n_codebook: int = 1, lfq_bias: bool = True,
                 lfq_frac_sample: float = 1., lfq_commit_weight: float = 0.25, lfq_entropy_weight: float = 0.1,
                 lfq_diversity_weight: float = 1., quant_loss_weight: float = 1.) -> None:
        super().__init__()
        if n_codebook != 1:
            # the reference's quantiser here projects from 2^d_codebook * n_codebook inputs and cannot run; this
            # class feeds it the d_codebook-wide output of to_act, which n_codebook > 1 codebooks cannot split
            raise NotImplementedError(f'LatentAction supports n_codebook = 1 only (got {n_codebook}): the action '
                                      f'head to_act emits d_codebook = {d_codebook} values per frame, one codebook')
        if isinstance(inp_shape, int):
            inp_shape = (inp_shape, inp_shape)
        self.proj_in = CausalConv3d(inp_channels, out_channels=n_embd, kernel_size=ker_size)
        self.proj_out = CausalConv3d(n_embd, out_channels=inp_channels, kernel_size=ker_size)
        self.proj_out.out_f32 = True                            # feeds mse_loss
        self.enc_layers, self.enc_ext = parse_blueprint(enc_desc)
        self.dec_layers, self.dec_ext = parse_blueprint(dec_desc)
        enc_fact = prod(enc.factor for enc in self.enc_layers if isinstance(enc, (Downsample, Upsample)))
        dec_fact = prod(dec.factor for dec in self.dec_layers if isinstance(dec, (Downsample, Upsample)))
        assert enc_fact * dec_fact == 1, 'The product of the space-time up/down factors must be 1.'
        self.to_act = nn.Sequential(nn.Identity(), _ToActLinear(int(n_embd * enc_fact * prod(inp_shape)), d_codebook))
        self.quant = LookupFreeQuantization(
            codebook_dim=d_codebook, num_codebook=n_codebook, input_dim=d_codebook * n_codebook, use_bias=lfq_bias,
            frac_sample=lfq_frac_sample, commit_weight=lfq_commit_weight, entropy_weight=lfq_entropy_weight,
            diversity_weight=lfq_diversity_weight)
        self.d_codebook, self.n_codebook = d_codebook, n_codebook
        self.quant_loss_weight = quant_loss_weight

    def sample(self, idxs: Tensor) -> Tensor:
        return self.quant.codebook[idxs]

    def encode(self, video: Tensor, mask: Tensor | None = None, transpose: bool = False):
        video = self.proj_in(video)
        for enc in self.enc_layers:
            video = enc(video, mask=mask)
        act = self.to_act(video)
        (act, idxs), q_loss = self.quant(act, transpose=transpose)
        return (act, idxs, video), q_loss

    def decode(self, video: Tensor, q_act: Tensor) -> Tensor:
        for dec, has_ext in zip(self.dec_layers, self.dec_ext):
            video = dec(video, cond=(None, q_act if has_ext else None))
        return self.proj_out(video)

    def forward(self, video: Tensor, mask: Tensor | None = None):
        (act, idxs, enc_video), q_loss = self.encode(video, mask=mask)
        recon = self.decode(enc_video, act)
        rec_loss = ops.mse_loss(recon, video)
        loss = rec_loss + q_loss * self.quant_loss_weight
        return idxs, loss, (rec_loss, q_loss)
