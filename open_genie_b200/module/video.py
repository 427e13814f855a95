"""Video building blocks — same class names, constructor kwargs and state_dict keys as the reference's
genie/module/video.py, but every forward runs hand-written sm_90a kernels through the C ABI.

state_dict compatibility: conv weights are ordinary (Cout, Cin, kt, kh, kw) fp32 parameters (stored in
channels_last_3d memory so their bytes ARE the kernels' [Cout][tap][Cin] operand order); the bf16 operand
copy is a non-persistent buffer refreshed whenever the parameter changes.
"""
from __future__ import annotations

import math
import weakref
from abc import ABC
from typing import Tuple

import torch
import torch.nn as nn
from torch import Tensor

from .. import ops
from ..utils import default, exists


# id(weight Parameter) -> Conv3dParams that owns it; lets FusedAdamW refresh the packed bf16 operand in its own pass
CONV_REGISTRY = weakref.WeakValueDictionary()


def _triple(v):
    return (v, v, v) if isinstance(v, int) else tuple(v)


class Conv3dParams(nn.Module):
    """Parameter holder with nn.Conv3d's state_dict layout ('weight', 'bias') plus the packed bf16 operand."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=(1, 1, 1), causal=True, bias=True):
        super().__init__()
        kernel_size, stride = _triple(kernel_size), _triple(stride)
        self.geom = ops.ConvGeom(in_channels, out_channels, kernel_size, stride, causal=causal)
        w = torch.empty(out_channels, in_channels, *kernel_size)
        # same default init as nn.Conv3d (kaiming_uniform(a=sqrt(5)) / uniform bias)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        self.weight = nn.Parameter(w.contiguous(memory_format=torch.channels_last_3d))
        if bias:
            bound = 1 / math.sqrt(in_channels * math.prod(kernel_size))
            self.bias = nn.Parameter(torch.empty(out_channels).uniform_(-bound, bound))
        else:
            self.register_parameter('bias', None)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = kernel_size, stride
        self._packed = None
        self._packed_key = None
        self._extra = None          # optional fused 1x1x1 shortcut (Conv3dParams)
        self._fused_into = None     # weakref to the conv whose operand matrix carries this shortcut
        CONV_REGISTRY[id(self.weight)] = self

    def __setstate__(self, state):
        """copy.deepcopy / pickle (EMA copies, ddp_spawn): the copy owns NEW Parameter objects, so it must register
        itself (FusedAdamW finds the bf16 operand of a weight through CONV_REGISTRY) and rebuild its packed operand;
        the owning block re-links fused shortcuts (a deep-copied weakref still points at the ORIGINAL module)."""
        super().__setstate__(state)
        self._packed = None
        self._packed_key = None
        object.__setattr__(self, '_fused_into', None)
        CONV_REGISTRY[id(self.weight)] = self

    def fuse_shortcut(self, other: 'Conv3dParams'):
        """Append `other` (a 1x1x1 conv on a second input) as extra K columns of the packed operand, so
        main(x) + res(x) (genie/module/video.py:648) is ONE implicit GEMM with one accumulator."""
        assert other.kernel_size == (1, 1, 1) and other.out_channels == self.out_channels and self.geom.direct
        object.__setattr__(self, '_extra', other)
        object.__setattr__(other, '_fused_into', weakref.ref(self))
        self._packed_key = None

    def packed(self) -> Tensor:
        """bf16 [Cout][ld] operand matrix: main taps (tap-major, channel-minor), then the fused shortcut."""
        w = self.weight
        e = self._extra
        key = (w.data_ptr(), w._version, w.device) + ((e.weight.data_ptr(), e.weight._version) if e is not None else ())
        if self._packed is None or self._packed_key != key:
            ld = self.geom.kpad + (e.in_channels if e is not None else 0)
            if self._packed is None or self._packed.shape[1] != ld or self._packed.device != w.device:
                self._packed = torch.zeros((self.out_channels, ld), dtype=torch.bfloat16, device=w.device)
            ops.pack_weight(w, self._packed, 0, self.geom.cin_pad)
            if e is not None:
                ops.pack_weight(e.weight, self._packed, self.geom.kpad)
            self._packed_key = key
        return self._packed

    def bf16_target(self):
        """(packed operand matrix, column offset) that must be rewritten whenever self.weight changes.
        FusedAdamW updates weights through raw pointers (torch's version counter does not move), so it
        writes the bf16 copy itself, in the same pass."""
        owner = self._fused_into() if self._fused_into is not None else None
        if owner is not None:
            return owner.packed(), owner.geom.kpad
        if self.geom.padded:     # every tap's Cin channels sit at a pitch of cin_pad in the packed operand
            return self.packed(), 0, self.in_channels, self.geom.cin_pad
        return self.packed(), 0

    def forward(self, x: Tensor, x2: Tensor | None = None, out_f32: bool = False) -> Tensor:
        ops._require_cuda(x, 'conv input')
        if not self.weight.is_cuda:
            raise RuntimeError('open_genie_b200: module parameters must be on a CUDA device (no CPU path); '
                               'call .cuda() / .to("cuda") first')
        e = self._extra
        assert (x2 is None) or (e is not None), 'second input given but no fused shortcut registered'
        if e is not None and x2 is not None:
            return ops.conv3d(x, self.weight, self.bias, self.packed(), self.geom, out_f32, x2, e.weight, e.bias)
        return ops.conv3d(x, self.weight, self.bias, self.packed(), self.geom, out_f32)


def _causal_space_pads(padding, kernel_size):
    """The (height, width) pads CausalConv3d derives from `padding` (genie/module/video.py:144-157): an int or None is
    used for both, otherwise entries 0 and 1 are the height and width pads and further entries are ignored; None means
    (k - 1) // 2. Returns None for a `padding` the reference would not accept."""
    if padding is None or isinstance(padding, int):
        padding = (padding, padding)
    if not isinstance(padding, (tuple, list)) or len(padding) < 2:
        return None
    _, kh, kw = kernel_size
    return (default(padding[0], (kh - 1) // 2), default(padding[1], (kw - 1) // 2))


class CausalConv3d(nn.Module):
    """3-D causal convolution: time padded on the left only. Mirrors genie/module/video.py:106-200
    (state_dict keys 'conv3d.weight', 'conv3d.bias'). pad_mode='constant' and dilation 1 only. `padding` is accepted
    when it resolves to the default spatial pads, (kh - 1) // 2 and (kw - 1) // 2, which are the pads the kernels
    implement."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size, stride=(1, 1, 1), dilation=(1, 1, 1),
                 padding=None, pad_mode: str = 'constant', **kwargs):
        super().__init__()
        if _triple(dilation) != (1, 1, 1):
            raise NotImplementedError('CausalConv3d: dilation != 1 is outside the hot-path scope')
        k = _triple(kernel_size)
        if pad_mode != 'constant' or _causal_space_pads(padding, k) != ((k[1] - 1) // 2, (k[2] - 1) // 2):
            raise NotImplementedError('CausalConv3d: only constant padding with the default spatial pads '
                                      '((k - 1) // 2) is implemented')
        self.conv3d = Conv3dParams(in_channels, out_channels, kernel_size, stride, causal=True,
                                   bias=kwargs.get('bias', True))
        self.in_channels, self.out_channels = in_channels, out_channels
        self.out_f32 = False        # set by VideoTokenizer on the layers that feed a loss

    def forward(self, inp: Tensor) -> Tensor:
        return self.conv3d(inp, out_f32=self.out_f32)

    @property
    def inp_dim(self) -> int:
        return self.in_channels

    @property
    def out_dim(self) -> int:
        return self.out_channels


class Upsample(nn.Module, ABC):
    """genie/module/video.py:58-80"""

    def __init__(self, time_factor: int = 1, space_factor: int = 1) -> None:
        super().__init__()
        self.time_factor, self.space_factor = time_factor, space_factor
        self.go_up = None

    @property
    def factor(self):
        return self.time_factor * (self.space_factor ** 2)

    def forward(self, inp: Tensor, **kwargs) -> Tensor:
        return self.go_up(inp)


class Downsample(nn.Module, ABC):
    """genie/module/video.py:82-104"""

    def __init__(self, time_factor: int = 1, space_factor: int = 1) -> None:
        super().__init__()
        self.time_factor, self.space_factor = time_factor, space_factor
        self.go_down = None

    @property
    def factor(self):
        return self.time_factor * (self.space_factor ** 2)

    def forward(self, inp: Tensor, **kwargs) -> Tensor:
        return self.go_down(inp)


class SpaceTimeDownsample(Downsample):
    """Strided CausalConv3d — genie/module/video.py:457-483 (key 'go_down.conv3d.*')."""

    def __init__(self, in_channels: int, kernel_size, out_channels: int | None = None, time_factor: int = 2,
                 space_factor: int = 2, **kwargs) -> None:
        super().__init__(time_factor=1 / time_factor, space_factor=1 / space_factor)
        self.go_down = CausalConv3d(in_channels, default(out_channels, in_channels), kernel_size=_triple(kernel_size),
                                    stride=(time_factor, space_factor, space_factor), **kwargs)
        self.in_channels, self.out_channels = in_channels, default(out_channels, in_channels)


class _PixelShuffle3d(nn.Module):
    def __init__(self, p, q, r):
        super().__init__()
        self.p, self.q, self.r = p, q, r

    def forward(self, x):
        return ops.pixel_shuffle3d(x, self.p, self.q, self.r)


class DepthToSpaceTimeUpsample(Upsample):
    """CausalConv3d to C*tf*sf^2 channels followed by the depth-to-space-time rearrange —
    genie/module/video.py:379-430 (key 'go_up.0.conv3d.*')."""

    def __init__(self, in_channels: int, out_channels: int | None = None, time_factor: int = 2,
                 space_factor: int = 2, kernel_size=1) -> None:
        super().__init__(time_factor=time_factor, space_factor=space_factor)
        out_channels = default(out_channels, in_channels)
        self.go_up = nn.Sequential(
            CausalConv3d(in_channels, out_channels * time_factor * space_factor ** 2, kernel_size=kernel_size),
            _PixelShuffle3d(time_factor, space_factor, space_factor),
        )
        self.in_channels, self.out_channels = in_channels, out_channels

    def forward(self, inp: Tensor, **kwargs) -> Tensor:
        return self.go_up(inp)

    @property
    def inp_dim(self):
        return self.in_channels

    @property
    def out_dim(self):
        return self.out_channels


class BlurPooling3d(nn.Module):
    """Anti-aliased strided pooling — genie/module/video.py:487-537. The reference repeats one normalised Pascal kernel
    over a conv with `num_groups` groups, so output channel o of group g = o // (out_channels / num_groups) is
    blur(sum of input group g); with num_groups == 1 every output channel is blur(sum_c x_c). That is what the kernels
    compute. Time is padded symmetrically by (k - 1) // 2 like space, also inside a causal VideoResidualBlock, as in
    the reference: the pooling is not causal. Buffer 'blur' is kept for state_dict parity."""

    def __init__(self, in_channels: int, kernel_size, out_channels: int | None = None, time_factor: int = 2,
                 space_factor=2, num_groups: int = 1, **kwargs) -> None:
        super().__init__()
        kernel_size = _triple(kernel_size)
        if len(set(kernel_size)) != 1 or kwargs:
            raise NotImplementedError('BlurPooling3d: cubic kernels only')
        if num_groups < 1 or (out_channels is not None and out_channels % num_groups):
            raise ValueError(f'BlurPooling3d: out_channels={out_channels} must be divisible by num_groups={num_groups}')
        if isinstance(space_factor, int):
            space_factor = (space_factor, space_factor)
        k = kernel_size[0]
        row = torch.tensor([math.comb(k - 1, i) for i in range(k)], dtype=torch.float32)
        ker = row[:, None, None] * row[None, :, None] * row[None, None, :]
        self.register_buffer('blur', ker / ker.sum())
        self.k = k
        self.stride = (time_factor, *space_factor)
        self.num_groups = num_groups
        self.out_channels = out_channels

    def forward(self, inp: Tensor) -> Tensor:
        cout = default(self.out_channels, inp.shape[1])
        if inp.shape[1] % self.num_groups or cout % self.num_groups:
            raise ValueError(f'BlurPooling3d: {inp.shape[1]} input and {cout} output channels must be divisible by '
                             f'num_groups={self.num_groups}')
        return ops.blurpool3d(inp, self.k, self.stride, cout, self.num_groups)


class _GNParams(nn.GroupNorm):
    """nn.GroupNorm as parameter holder (keys 'weight', 'bias'); forward runs the fused kernel."""
    act = 'none'

    def forward(self, x: Tensor) -> Tensor:
        return ops.group_norm_act(x, self.weight, self.bias, self.num_groups, self.eps, self.act)


class _Slot(nn.Identity):
    """Keeps nn.Sequential indices aligned with the reference (activation / Identity positions)."""


def _conv_params(m: nn.Module) -> Conv3dParams:
    return m.conv3d if isinstance(m, CausalConv3d) else m


def _handed_over_sums(x: Tensor):
    """The GroupNorm(1) sums a fused block stored on its output x, if they still describe x: not after an in-place
    edit of x (its version moved), and not after a step boundary of the zero arena that holds them (they may have
    been zeroed). None means the consumer computes them itself. Inference tensors have no version counter, so
    inference_mode forwards never hand sums over."""
    handed = getattr(x, '_og_gn_sums', None)
    if handed is None or x.is_inference():
        return None
    sums, version, arena, generation = handed
    if x._version != version or (arena is not None and arena.generation != generation):
        return None
    return sums


class VideoResidualBlock(nn.Module):
    """GN -> act -> conv -> GN -> act -> conv, plus an (always present) 1x1x1 conv shortcut —
    genie/module/video.py:539-656. state_dict keys: main.{0,4}.{weight,bias}, main.{2,6}.{weight,bias},
    res.1.{weight,bias}; with use_causal=True every conv is a CausalConv3d (main.{2,6}.conv3d.*, res.1.conv3d.*).

    use_causal=True pads time by kt - 1 frames in front and none behind. The block is still not strictly causal, in the
    reference too: GroupNorm statistics span all frames, and the blur pooling of `downsample` pads time symmetrically.
    The reference passes padding=((kt-1)//2, (kh-1)//2, (kw-1)//2) to its CausalConv3d, which reads entries 0 and 1 as
    the height and width pads; kernels where that differs from the default pads change H and W there, and raise here.

    GPU execution: each GN+act is one statistics pass + one fused apply pass, and the second conv, the
    shortcut conv and the residual add are a single implicit GEMM (the shortcut's K columns are appended
    to the main conv's operand matrix)."""

    def __init__(self, in_channels: int, out_channels: int | None = None, kernel_size=3, num_groups: int = 1,
                 pad_mode: str = 'constant', downsample=None, use_causal: bool = False, use_norm: bool = True,
                 use_blur: bool = True, act_fn: str = 'swish') -> None:
        super().__init__()
        if isinstance(downsample, int):
            downsample = (downsample, downsample)
        if exists(downsample) and not use_blur:
            raise NotImplementedError('VideoResidualBlock(downsample=..., use_blur=False) does not construct in the '
                                      'reference (it passes num_groups to nn.Conv3d)')
        if act_fn not in ('swish', 'silu', 'leaky', 'relu') or not use_norm or pad_mode != 'constant':
            raise NotImplementedError('VideoResidualBlock: GroupNorm + SiLU / LeakyReLU / ReLU blocks are implemented')
        self.act_fn = 'silu' if act_fn == 'swish' else act_fn
        kernel_size = _triple(kernel_size)
        if use_causal and len({(k - 1) // 2 for k in kernel_size}) != 1:
            raise NotImplementedError(
                f'VideoResidualBlock(use_causal=True, kernel_size={kernel_size}): the reference pads height by '
                f'(kt - 1) // 2 and width by (kh - 1) // 2 (its CausalConv3d reads the padding tuple from the time '
                f'entry), which changes H and W and breaks its residual add; only kernels with equal (k - 1) // 2 in '
                f'all three dimensions are implemented')
        out_channels = default(out_channels, in_channels)
        if use_causal:
            conv = lambda ci, co, k: CausalConv3d(ci, co, k)
        else:
            conv = lambda ci, co, k: Conv3dParams(ci, co, k, causal=False)
        tf, sf = downsample if exists(downsample) else (None, None)
        down = (lambda c: BlurPooling3d(c, kernel_size, time_factor=tf, space_factor=sf, num_groups=num_groups)) \
            if exists(downsample) else (lambda c: _Slot())
        self.res = nn.Sequential(down(in_channels), conv(in_channels, out_channels, 1))
        self.main = nn.Sequential(
            _GNParams(num_groups, in_channels), _Slot(), conv(in_channels, out_channels, kernel_size), down(out_channels),
            _GNParams(num_groups, out_channels), _Slot(), conv(out_channels, out_channels, kernel_size),
        )
        self.has_down = exists(downsample)
        self.use_causal = use_causal
        self.main[0].act = self.main[4].act = self.act_fn
        _conv_params(self.main[6]).fuse_shortcut(_conv_params(self.res[1]))
        self.inp_channels, self.out_channels = in_channels, out_channels
        self.in_channels = in_channels

    def __setstate__(self, state):
        super().__setstate__(state)
        # re-link inside the copy (see Conv3dParams.__setstate__)
        _conv_params(self.main[6]).fuse_shortcut(_conv_params(self.res[1]))

    def forward(self, inp: Tensor) -> Tensor:
        fusable = all((c // self.main[0].num_groups) % 8 == 0 for c in (self.inp_channels, self.out_channels))
        c1, c2, cr = _conv_params(self.main[2]), _conv_params(self.main[6]), _conv_params(self.res[1])
        if not self.has_down and inp.is_cuda and fusable:
            # whole block as one autograd node: GroupNorm statistics / backward reductions come out of the GEMM
            # epilogues, the shortcut gradient is added inside the last apply pass. The statistics of the output
            # ride along on the tensor so that the next block's first GroupNorm needs no pass of its own.
            g1, g2 = self.main[0], self.main[4]
            ops._require_cuda(c1.weight, 'module parameters')
            sums = _handed_over_sums(inp) if g1.num_groups == 1 else None
            y, y_sums = ops.residual_block(inp, sums, g1.weight, g1.bias, c1.weight, c1.bias, g2.weight, g2.bias,
                                           c2.weight, c2.bias, cr.weight, cr.bias, c1.packed(), c2.packed(), c1.geom,
                                           c2.geom, g1.num_groups, g1.eps, act=self.act_fn)
            if not y.is_inference():
                arena = ops.current_arena()
                if arena is not None and arena.locate(y_sums) is None:
                    arena = None
                y._og_gn_sums = (y_sums, y._version, arena, arena.generation if arena is not None else None)
            return y
        h = self.main[0](inp)                # GN + act (fused)
        h = c1(h)                            # conv k3
        skip = inp
        if self.has_down:                    # anti-aliased down-sampling of both branches (video.py:589-621)
            h = self.main[3](h)
            skip = self.res[0](inp)
        h = self.main[4](h)                  # GN + act (fused)
        return c2(h, x2=skip)                # conv k3 (+) 1x1x1 shortcut (+) add : one kernel

    @property
    def inp_dim(self):
        return self.inp_channels

    @property
    def out_dim(self):
        return self.out_channels
