"""2-D image modules of the reference's registry (genie/module/image.py) that the hot path can reach by blueprint
name. A (B, C, H, W) image is handled as an NHWC bf16 tensor, i.e. the T = 1 case of the NDHWC kernels."""
from __future__ import annotations

import math
from typing import Tuple

import torch
import torch.nn as nn
from torch import Tensor

from .. import _lib, ops


class _BlurPool2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k: int, stride: Tuple[int, int], pad: int):
        ops._require_cuda(x, 'blur_pool input')
        B, C, H, W = x.shape
        xi = x.detach().permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()            # NHWC rows
        sh, sw = stride
        Ho, Wo = (H + 2 * pad - k) // sh + 1, (W + 2 * pad - k) // sw + 1
        y = torch.empty((B, Ho, Wo, C), dtype=torch.bfloat16, device=x.device)
        scratch = torch.empty(B * H * W, dtype=torch.float32, device=x.device)
        _lib.call('og_blurpool2d', xi.data_ptr(), y.data_ptr(), scratch.data_ptr(), 0, B, H, W, C, C, k, sh, sw, pad,
                  ops._stream())
        ctx.cfg = (B, C, H, W, k, sh, sw, pad, Ho, Wo, x.dtype)
        return y.permute(0, 3, 1, 2).to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        B, C, H, W, k, sh, sw, pad, Ho, Wo, dtype = ctx.cfg
        dyi = dy.detach().permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()
        dx = torch.empty((B, H, W, C), dtype=torch.bfloat16, device=dy.device)
        scratch = torch.empty(B * Ho * Wo, dtype=torch.float32, device=dy.device)
        _lib.call('og_blurpool2d', dyi.data_ptr(), dx.data_ptr(), scratch.data_ptr(), 1, B, H, W, C, C, k, sh, sw, pad,
                  ops._stream())
        return dx.permute(0, 3, 1, 2).to(dtype), None, None, None


class BlurPooling2d(nn.Module):
    """Anti-aliased strided pooling of images — genie/module/image.py:43-85, registry name 'blur_pool'
    (genie/module/__init__.py:33). Same constructor, same 'blur' buffer, same quirky padding `(k-1) // stride`.
    With num_groups == 1 the reference's repeated kernel makes every output channel blur(sum_c x_c) (SURVEY.md §8 a6);
    that is what og_blurpool2d computes. Returns a (B, C, Ho, Wo) tensor of the input's dtype."""

    def __init__(self, kernel_size, stride=2, num_groups: int = 1, **kwargs) -> None:
        super().__init__()
        ker = (kernel_size, kernel_size) if isinstance(kernel_size, int) else tuple(kernel_size)
        strd = (stride, stride) if isinstance(stride, int) else tuple(stride)
        if ker[0] != ker[1] or num_groups != 1 or kwargs:
            raise NotImplementedError('BlurPooling2d: square kernels and num_groups == 1 only')
        row = torch.tensor([math.comb(ker[0] - 1, i) for i in range(ker[0])], dtype=torch.float32)
        k2 = row[:, None] * row[None, :]
        self.register_buffer('blur', k2 / k2.sum())
        self.k, self.stride, self.num_groups = ker[0], strd, num_groups
        pad = ((ker[0] - 1) // strd[0], (ker[1] - 1) // strd[1])
        if pad[0] != pad[1]:
            raise NotImplementedError('BlurPooling2d: equal strides only')
        self.padding = pad

    def forward(self, inp: Tensor) -> Tensor:
        if inp.shape[1] % 8 != 0:
            raise NotImplementedError('BlurPooling2d kernels need a channel count that is a multiple of 8')
        return _BlurPool2dFn.apply(inp, self.k, self.stride, self.padding[0])


# ------------------------------------------------------------------------------------------------
# 2-D convolutional blocks of the frame discriminator (genie/module/image.py:86-161). An image batch (n, c, h, w) runs
# as the T = 1 case of the NDHWC kernels: internally every tensor here is the 5-D internal format (n, c, 1, h, w).
# ------------------------------------------------------------------------------------------------
from .video import Conv3dParams, _GNParams, _Slot      # noqa: E402


class Conv2dParams(Conv3dParams):
    """nn.Conv2d parameter layout in the state_dict (weight (Cout, Cin, kh, kw)), executed as a (1, kh, kw) 3-D
    convolution with symmetric padding (k-1)//2 — the `padding=1` / `kernel_size=1` convolutions of image.py."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, bias=True):
        k = (kernel_size, kernel_size) if isinstance(kernel_size, int) else tuple(kernel_size)
        s = (stride, stride) if isinstance(stride, int) else tuple(stride)
        strided = s != (1, 1)
        # a strided convolution goes through the CausalConv3d geometry, which coincides with nn.Conv2d's for k = 1
        assert not strided or k == (1, 1), 'strided 2-D convolutions are only used with kernel_size = 1'
        super().__init__(in_channels, out_channels, (1,) + k, stride=(1,) + s, causal=strided, bias=bias)

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        w = destination[prefix + 'weight']
        destination[prefix + 'weight'] = w.squeeze(2) if w.dim() == 5 else w

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        k = prefix + 'weight'
        if k in state_dict and state_dict[k].dim() == 4:
            state_dict = dict(state_dict)
            state_dict[k] = state_dict[k].unsqueeze(2)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


class _SpaceToDepth(nn.Module):
    def __init__(self, factor: int):
        super().__init__()
        self.factor = factor

    def forward(self, x):
        return ops.space_to_depth3d(x, 1, self.factor, self.factor)


class SpaceDownsample(nn.Module):
    """Rearrange('b c (h p) (w q) -> b (c p q) h w') + Conv2d(in_dim * factor^2, in_dim, 1) — genie/module/image.py:86-104
    (keys go_up.1.{weight,bias}; the attribute really is called `go_up` in the reference)."""

    def __init__(self, in_dim: int, factor: int = 2) -> None:
        super().__init__()
        self.go_up = nn.Sequential(_SpaceToDepth(factor), Conv2dParams(in_dim * factor ** 2, in_dim, 1))

    def forward(self, inp: Tensor, residual: Tensor | None = None) -> Tensor:
        c = self.go_up[1]
        return ops.conv3d(self.go_up[0](inp), c.weight, c.bias, c.packed(), c.geom, residual=residual)


class ImageResidualBlock(nn.Module):
    """GN -> LeakyReLU -> Conv2d -> GN -> LeakyReLU -> Conv2d [-> SpaceDownsample]  +  Conv2d(k=1, stride=downsample)
    — genie/module/image.py:106-161. state_dict keys main.{0,3}.* (GroupNorm), main.{2,5}.* (Conv2d),
    main.6.go_up.1.*, res.*. Without down-sampling the whole block is the fused residual-block node (GroupNorm
    statistics in the GEMM epilogues, shortcut as extra K columns); with it the shortcut's strided 1x1 convolution is
    added inside the epilogue of the SpaceDownsample convolution."""

    def __init__(self, inp_channel: int, out_channel: int | None = None, kernel_size=3, padding=1, num_groups: int = 1,
                 downsample: int | None = None) -> None:
        super().__init__()
        k = (kernel_size, kernel_size) if isinstance(kernel_size, int) else tuple(kernel_size)
        pd = (padding, padding) if isinstance(padding, int) else tuple(padding)
        if pd != ((k[0] - 1) // 2, (k[1] - 1) // 2):
            raise NotImplementedError('ImageResidualBlock: only "same" padding is implemented')
        self.res = Conv2dParams(inp_channel, out_channel, 1, stride=downsample if downsample else 1) \
            if out_channel is not None else nn.Identity()
        out_channel = out_channel if out_channel is not None else inp_channel
        layers = [_GNParams(num_groups, inp_channel), _Slot(), Conv2dParams(inp_channel, out_channel, k),
                  _GNParams(num_groups, out_channel), _Slot(), Conv2dParams(out_channel, out_channel, k)]
        if downsample:
            layers.append(SpaceDownsample(out_channel, downsample))
        self.main = nn.Sequential(*layers)
        self.main[0].act = self.main[3].act = 'leaky'
        self.downsample = downsample
        self.inp_channel, self.out_channel = inp_channel, out_channel
        self._fusable = (not downsample) and isinstance(self.res, Conv2dParams)
        if self._fusable:
            self.main[5].fuse_shortcut(self.res)

    def __setstate__(self, state):
        super().__setstate__(state)
        if self._fusable:
            self.main[5].fuse_shortcut(self.res)

    def forward(self, inp: Tensor) -> Tensor:
        g1, c1, g2, c2 = self.main[0], self.main[2], self.main[3], self.main[5]
        G = g1.num_groups
        if self._fusable and (self.inp_channel % 64 or self.out_channel % 64):
            raise NotImplementedError(f'ImageResidualBlock({self.inp_channel}, {self.out_channel}): a block with a 1x1 '
                                      f'shortcut runs it as extra K columns of the last convolution, which needs '
                                      f'channel counts that are multiples of 64')
        if self._fusable and all((c // G) % 8 == 0 for c in (self.inp_channel, self.out_channel)):
            y, _ = ops.residual_block(inp, None, g1.weight, g1.bias, c1.weight, c1.bias, g2.weight, g2.bias, c2.weight,
                                      c2.bias, self.res.weight, self.res.bias, c1.packed(), c2.packed(), c1.geom, c2.geom,
                                      G, g1.eps, act='leaky')
            return y
        h = c1(g1(inp))
        h = g2(h)
        if self._fusable:        # the shortcut's only bf16 weights are main[5]'s extra K columns (FusedAdamW writes those)
            return c2(h, x2=inp)
        skip = self.res(inp) if isinstance(self.res, Conv2dParams) else inp
        if self.downsample:
            h = c2(h)
            return self.main[6](h, residual=skip)
        return ops.conv3d(h, c2.weight, c2.bias, c2.packed(), c2.geom, residual=skip)
