"""GAN critics of the tokenizer objective — mirrors genie/module/discriminator.py:17-221 (same constructors, same
state_dict keys: proj_in.*, core.N.0.{main,res}.*, to_logits.{0,3}.*) on the CUDA kernels."""
from __future__ import annotations

from itertools import pairwise
from math import prod
from typing import Tuple

import torch
import torch.nn as nn
from torch import Tensor

from .. import ops
from .image import Conv2dParams, ImageResidualBlock


class _LogitsHead(nn.Module):
    """nn.Linear(latent_dim, 1) on 'b c h w -> b (c h w)' (discriminator.py:95-101). Activations are channels-last, so the
    weight keeps the reference's (c, h, w) column order in the state_dict and is permuted when its bf16 operand is cast;
    the single output row is padded to 8 for the GEMM kernel."""

    def __init__(self, latent_dim: int) -> None:
        super().__init__()
        lin = nn.Linear(latent_dim, 1)
        self.weight = nn.Parameter(lin.weight.detach().clone())
        self.bias = nn.Parameter(lin.bias.detach().clone())

    def forward(self, x: Tensor) -> Tensor:                       # internal (n, C, 1, h, w) -> (n,)
        n, C, T, h, w = x.shape
        rows = x.permute(0, 2, 3, 4, 1)
        if rows.dtype != torch.bfloat16 or not rows.is_contiguous():
            rows = rows.to(torch.bfloat16).contiguous()
        wp = self.weight.view(1, C, T * h, w).permute(0, 2, 3, 1).reshape(1, T * h * w * C)
        wp = torch.cat([wp, wp.new_zeros(7, wp.shape[1])], 0)
        packed = wp.detach().to(torch.bfloat16).contiguous()
        y = ops.linear_rows(rows.reshape(n, T * h * w * C), wp.contiguous(), None, packed, out_f32=True)
        return y[:, 0] + self.bias


class FrameDiscriminator(nn.Module):
    """genie/module/discriminator.py:17-114. `use_attn=True` is not implemented (its SpatialAttention(d_inp=out_dim,
    n_head=4, d_head=32) fails the reference's own LayerNorm shape check unless out_dim == 128)."""

    def __init__(self, inp_size, model_dim: int = 64, dim_mults: Tuple[int, ...] = (1, 2, 4),
                 down_step: Tuple[int | None, ...] = (None, 2, 2), inp_channels: int = 3, kernel_size=3, num_groups: int = 1,
                 num_heads: int = 4, dim_head: int = 32, use_attn: bool = False, use_blur: bool = True,
                 act_fn: str = 'leaky') -> None:
        super().__init__()
        if use_attn:
            raise NotImplementedError('FrameDiscriminator(use_attn=True) is outside the hot-path scope')
        if isinstance(inp_size, int):
            inp_size = (inp_size, inp_size)
        dims = [model_dim * mult for mult in dim_mults]
        assert len(dims) == len(down_step), 'Dimension and downsample steps must match.'
        self.proj_in = Conv2dParams(inp_channels, model_dim, 3)
        self.core = nn.ModuleList([])
        out_dim = model_dim
        for (inp_dim, out_dim), down in zip(pairwise(dims), down_step):          # NB: zip stops at len(dims) - 1 blocks
            self.core.append(nn.ModuleList([
                ImageResidualBlock(inp_dim, out_dim, downsample=down, num_groups=num_groups, kernel_size=kernel_size),
                nn.ModuleList([nn.Identity(), nn.Identity()])]))
            inp_size = tuple(map(lambda x: x // (down or 1), inp_size))
        latent_dim = out_dim * prod(inp_size)
        self.to_logits = nn.Sequential(Conv2dParams(out_dim, out_dim, 3), nn.Identity(), nn.Identity(),
                                       _LogitsHead(latent_dim), nn.Identity())

    def forward(self, image: Tensor) -> Tensor:
        """image: (n, c, h, w) in either format, or already internal (n, c, 1, h, w). Returns (n,) fp32 scores."""
        x = image if image.dim() == 5 else image.unsqueeze(2)
        c = self.proj_in
        out = ops.conv3d(x, c.weight, c.bias, c.packed(), c.geom)
        for res, _attn in self.core:
            out = res(out)
            # `out = attn(out) + out; out = ff(out) + out` with Identity attn / ff (discriminator.py:76-79, 107-111): x4
            out = ops.activation(out, 'none', 4.0)
        c = self.to_logits[0]
        out = ops.conv3d(out, c.weight, c.bias, c.packed(), c.geom)
        out = ops.activation(out, 'leaky')
        return self.to_logits[3](out)


class VideoDiscriminator(nn.Module):
    """genie/module/discriminator.py:116-221 (`gan_discriminate='video'`): the 3-D critic — nn.Conv3d stem, VideoResidualBlocks
    with LeakyReLU and blur-pool down-sampling, the same x4 Identity quirk, Conv3d + LeakyReLU + Linear head.
    `use_causal=True` / `use_attn=True` / `use_blur=False` do not construct in the reference either and raise here."""

    def __init__(self, inp_size, model_dim: int = 64, dim_mults: Tuple[int, ...] = (1, 2, 4),
                 down_step=(None, 2, 2), inp_channels: int = 3, kernel_size=3, num_groups: int = 1, num_heads: int = 4,
                 dim_head: int = 32, act_fn: str = 'leaky', use_attn: bool = False, use_blur: bool = True,
                 use_causal: bool = False) -> None:
        super().__init__()
        if use_attn or use_causal or not use_blur:
            raise NotImplementedError('VideoDiscriminator: use_attn / use_causal / use_blur=False are outside the scope')
        from .video import Conv3dParams, VideoResidualBlock
        inp_size = tuple(inp_size)
        if len(inp_size) == 2:
            inp_size = (inp_size[0], inp_size[1], inp_size[1])
        dims = [model_dim * mult for mult in dim_mults]
        assert len(dims) == len(down_step), 'Dimension and downsample steps must match.'
        self.proj_in = Conv3dParams(inp_channels, model_dim, kernel_size, causal=False)
        self.core = nn.ModuleList([])
        out_dim = model_dim
        for (inp_dim, out_dim), down in zip(pairwise(dims), down_step):
            self.core.append(nn.ModuleList([
                VideoResidualBlock(inp_dim, out_dim, downsample=down, num_groups=num_groups, kernel_size=kernel_size,
                                   act_fn=act_fn, use_blur=use_blur, use_causal=use_causal),
                nn.ModuleList([nn.Identity(), nn.Identity()])]))
            d = down if down is not None else (1, 1, 1)
            if isinstance(d, int):
                d = (d, d, d)
            if len(d) == 2:
                d = (d[0], d[1], d[1])
            inp_size = tuple(x // y for x, y in zip(inp_size, d))
        latent_dim = out_dim * prod(inp_size)
        self.to_logits = nn.Sequential(Conv3dParams(out_dim, out_dim, 3, causal=False), nn.Identity(), nn.Identity(),
                                       _LogitsHead(latent_dim), nn.Identity())

    def forward(self, video: Tensor) -> Tensor:
        c = self.proj_in
        out = ops.conv3d(video, c.weight, c.bias, c.packed(), c.geom)
        for res, _attn in self.core:
            out = res(out)
            out = ops.activation(out, 'none', 4.0)        # Identity attn / ff: x + x, twice (discriminator.py:213-218)
        c = self.to_logits[0]
        out = ops.conv3d(out, c.weight, c.bias, c.packed(), c.geom)
        out = ops.activation(out, 'leaky')
        return self.to_logits[3](out)
