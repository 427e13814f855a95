"""Space-time attention — same class names, constructor kwargs and state_dict keys as the reference's
genie/module/attention.py, executed by the fused CUDA kernels (csrc/attention_rows.cu, flash_attn.cu,
conv3d_*.cu).

Attention runs in the HEAD-valid configuration (SURVEY.md §7 H6/H8): d_inp == n_head*d_head, so to_q / to_k / to_v /
to_out are Identity, q = k = v = LayerNorm(RoPE(x)); the one live conditioning path is the temporal one (latent action
-> K, V through `time_attn_kw={'key_dim': k}`). Anything else raises.
Head widths: d_head = 16, 64 or 128 (flash attention and the temporal kernels have all three; temporal attention at 16
and 128 runs the tiled kernels at every clip length). Space and time attention may use different widths when n_head * d_head
matches, e.g. SpaceTimeAttention(n_head=(2, 1), d_head=(64, 128)) or (n_head=(4, 1), d_head=(16, 64)); the FFN
GroupNorm takes the temporal head count.
Rotary embeddings: `embed=False` (SpaceTimeAttention: a bool or a (space, time) pair) replaces the RotaryEmbedding by
nn.Identity, as the reference does, so q = k = v = LayerNorm(x) and the state_dict has no embed.freq key; the row
pass is then og_ln_rows_fwd / bwd instead of the fused RoPE+LayerNorm pass. It combines with every option below.
Dropout: `dropout` (0 <= p < 1) drops attention probabilities as SDPA's dropout_p does, in both the spatial and the
temporal attention. Like the reference, which passes dropout_p to the functional SDPA, it drops in eval mode and under
no_grad too; set `module.dropout = 0` (read at every call) for deterministic inference. The masks come from Philox
seeds drawn from the CUDA generator (csrc/attn_dropout.cuh), so torch.manual_seed governs them.
Causality: `causal` is SDPA's is_causal, as in the reference. SpatialAttention(causal=True) masks the tokens after
each one in raster order (og_flash_attn_causal_*); TemporalAttention defaults to causal=False, like the reference and
the `time_attn` blueprint, and then attends over the whole clip (og_temporal_attn_bidir_*, the tiled kernels at every
T). SpaceTimeAttention keeps the reference's spatial causal=False and temporal causal=True.
The FFN is the reference's ForwardBlock: GroupNorm -> conv (-> GELU -> conv)* with `hid_dim` hidden widths, ending at
`d_out` channels (with transpose=True, where the skip becomes the 1x1x1 ffn_skip conv); `bias` gives every FFN conv a
bias. Hidden widths and d_out are multiples of 64.
state_dict keys: {space,temp}_attn.norm.{weight,bias}, {space,temp}_attn.embed.freq (with embed),
temp_attn.to_qkv.to_{k,v}.{weight[,bias]} (with key_dim), ffn.1.net.0.{weight,bias}, ffn.1.net.{i}.0.{weight[,bias]}
(i = 1 .. len(hid_dim) + 1), ffn_skip.{weight,bias} (d_out != n_head*d_head).
"""
from __future__ import annotations

from math import pi
from typing import Tuple

import torch
import torch.nn as nn
from torch import Tensor

from .. import ops
from ..utils import default, exists
from .video import Conv3dParams, _Slot


class RotaryEmbedding(nn.Module):
    """Holds the rotary frequencies exactly as the reference does (attention.py:17-46): '1d' =
    1/theta^(2i/dim), '2d' = linspace(1, max_freq/2, dim/2)*pi; `freq` is a (non-trainable) Parameter that
    lives in the state_dict. The rotation itself is fused into the RoPE+LayerNorm kernel."""

    def __init__(self, dim: int, kind: str = '1d', theta=10000, max_freq=10, learned_freq=False) -> None:
        super().__init__()
        if learned_freq:
            raise NotImplementedError('learned rotary frequencies are outside the hot-path scope')
        match kind:
            case '1d':
                freq = 1. / (theta ** (torch.arange(0, dim, 2)[:(dim // 2)].float() / dim))
            case '2d':
                freq = torch.linspace(1., max_freq / 2, dim // 2) * pi
            case _:
                raise NotImplementedError(f"RotaryEmbedding kind {kind!r} is not used on the hot path")
        self.freq = nn.Parameter(freq, requires_grad=False)


class Adapter(nn.Module):
    """Q/K/V adapter (attention.py:105-149): Identity where dims match, Linear(bias=False) for the K/V of a
    conditioning input of width key_dim."""

    def __init__(self, qry_dim: int, n_head: int, d_head: int, key_dim: int | None = None,
                 val_dim: int | None = None, bias: bool = False) -> None:
        super().__init__()
        key_dim = default(key_dim, qry_dim)
        val_dim = default(val_dim, key_dim)
        hid = n_head * d_head
        if qry_dim != hid:
            raise NotImplementedError('d_inp != n_head*d_head does not run in the reference either '
                                      '(LayerNorm dim mismatch, attention.py:179,220)')
        self.to_q = nn.Identity()
        self.to_k = nn.Linear(key_dim, hid, bias=bias) if key_dim != hid else nn.Identity()
        self.to_v = nn.Linear(val_dim, hid, bias=bias) if val_dim != hid else nn.Identity()
        self.n_head = n_head


class Attention(nn.Module):
    """Parameter layout of the reference's Attention (attention.py:154-239)."""
    rope_kind = None
    causal_default = False

    def __init__(self, n_head: int, d_head: int, d_inp: int | None = None, d_out: int | None = None, bias: bool = False,
                 embed: bool = True, scale: float | None = None, causal: bool = False, dropout: float = 0.0,
                 transpose: bool = False, **kwargs) -> None:
        super().__init__()
        hid = n_head * d_head
        self.d_inp = default(d_inp, hid)
        self.d_out = default(d_out, self.d_inp)
        if self.d_inp != hid or self.d_out != hid:
            raise NotImplementedError('only d_inp == d_out == n_head*d_head is valid at the reference HEAD')
        if not 0.0 <= dropout < 1.0:
            raise NotImplementedError(f'attention dropout must lie in [0, 1), not {dropout}')
        if d_head not in (16, 64, 128):
            raise NotImplementedError(f'the attention kernels take d_head = 16, 64 or 128, not {d_head}')
        self.norm = nn.LayerNorm(hid)
        # embed=False: no positional encoding, q = LayerNorm(x); nn.Identity as in the reference, so no embed.freq key
        self.embed = RotaryEmbedding(self.d_inp, kind=self.rope_kind) if embed else nn.Identity()
        self.to_qkv = Adapter(qry_dim=self.d_inp, n_head=n_head, d_head=d_head, bias=bias, **kwargs)
        self.n_head, self.d_head = n_head, d_head
        # reference precedence: default(scale, n_head * d_head ** -0.5)   (attention.py:195)
        self.scale = default(scale, n_head * d_head ** -0.5)
        self.causal = causal
        self.transpose = transpose
        self.dropout = dropout      # read at every forward call, as SDPA's dropout_p is (attention.py:229-234)

    def _rows(self, video: Tensor, transpose: bool | None) -> Tuple[Tensor, bool]:
        t = default(transpose, self.transpose)
        x = video.permute(0, 2, 3, 4, 1) if t else video            # -> (B, T, H, W, C), free for internal tensors
        return x, t

    @property
    def _freq(self) -> Tensor | None:
        """The rotary frequencies, or None without a rotary embedding (the attention functions then skip the rotation)."""
        return self.embed.freq if isinstance(self.embed, RotaryEmbedding) else None

    @staticmethod
    def _back(y: Tensor, t: bool) -> Tensor:
        return y.permute(0, 4, 1, 2, 3) if t else y


class SpatialAttention(Attention):
    """Self-attention over (h w) within each frame, 2-D rotary embedding (attention.py:241-307).
    forward returns attention(video) WITHOUT the skip, like the reference class."""
    rope_kind = '2d'

    def forward(self, video: Tensor, cond: Tensor | None = None, mask: Tensor | None = None,
                transpose: bool | None = None, _residual: bool = False) -> Tensor:
        if exists(cond) or exists(mask):
            raise NotImplementedError('spatial cond / mask are dead code at the reference HEAD (attention.py:290,296)')
        x, t = self._rows(video, transpose)
        y = ops.space_attention_res(x, self._freq, self.norm.weight, self.norm.bias, self.n_head, self.scale,
                                    self.norm.eps, self.dropout, self.causal)
        if not _residual:
            y = y - ops._rows_bf16(x)          # rarely used stand-alone path
        return self._back(y, t)


class TemporalAttention(Attention):
    """Self-attention over t for every pixel (causal with causal=True, bidirectional by default as in the reference),
    1-D rotary embedding; optional (B, T, key_dim) conditioning that provides K and V (attention.py:309-371)."""
    rope_kind = '1d'

    def forward(self, video: Tensor, cond: Tensor | None = None, mask: Tensor | None = None,
                transpose: bool | None = None, _residual: bool = False) -> Tensor:
        if exists(mask):
            raise NotImplementedError('SDPA forbids attn_mask together with is_causal (attention.py:229-234)')
        x, t = self._rows(video, transpose)
        kc = vc = None
        if exists(cond):
            c = cond.float()
            kc = self.to_qkv.to_k(c)            # (B, T, C): a few kFLOP of host-side plumbing (torch, autograd)
            vc = self.to_qkv.to_v(c)
        y = ops.time_attention_res(x, self._freq, self.norm.weight, self.norm.bias, self.n_head, self.scale,
                                   kc, vc, self.norm.eps, self.dropout, self.causal)
        if not _residual:
            y = y - ops._rows_bf16(x)
        return self._back(y, t)


class _FfnNet(nn.Module):
    """Mirror of ForwardBlock(in_dim, out_dim, hid_dim, block=nn.Conv3d, num_groups, bias, kernel_size, padding)
    (genie/module/misc.py:71-104): net = Sequential(GroupNorm, Sequential(Conv3d, GELU), ..., Sequential(Conv3d,
    Identity)) for state_dict keys net.0.*, net.{i}.0.{weight[,bias]}. The GELU slots hold no parameters: ops.ffn_res
    applies GELU with og_gelu_fwd / og_gelu_bwd."""

    def __init__(self, dim: int, out_dim: int, hid_dim: Tuple[int, ...], num_groups: int, kernel_size: int,
                 bias: bool) -> None:
        super().__init__()
        dims = (dim,) + hid_dim + (out_dim,)
        self.net = nn.Sequential(
            nn.GroupNorm(num_groups, dim),
            *[nn.Sequential(Conv3dParams(ci, co, kernel_size, causal=False, bias=bias),
                            _Slot() if i < len(dims) - 2 else nn.Identity())
              for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:]))],
        )


class SpaceTimeAttention(nn.Module):
    """x = space(x)+x ; x = time(x, cond)+x ; x = ffn(x)+x  (attention.py:373-474), three fused launches groups."""

    def __init__(self, n_head, d_head, d_inp: int | None = None, d_out: int | None = None, hid_dim=None,
                 bias: bool = False, embed=True, scale: float | None = None, dropout: float = 0.0,
                 kernel_size: int = 3, transpose: bool = False, time_attn_kw: dict = {}, space_attn_kw: dict = {}) -> None:
        super().__init__()
        if isinstance(n_head, int):
            n_head = (n_head, n_head)
        if isinstance(d_head, int):
            d_head = (d_head, d_head)
        if isinstance(embed, bool):
            embed = (embed, embed)
        if n_head[0] * d_head[0] != n_head[1] * d_head[1]:
            raise NotImplementedError('space and time widths must match')
        dim = n_head[1] * d_head[1]
        if exists(d_inp) and d_inp != dim:
            raise NotImplementedError('SpaceTimeAttention(d_inp != n_head*d_head) fails in the reference too: its '
                                      'spatial LayerNorm is built for n_head*d_head channels (attention.py:179,220)')
        d_out = default(d_out, dim)
        if d_out != dim and not transpose:
            raise NotImplementedError('SpaceTimeAttention(d_out != n_head*d_head) needs transpose=True: with '
                                      'transpose=False the reference applies its 1x1x1 ffn_skip conv to the '
                                      'channels-last tensor (attention.py:472) and fails')
        hid_dim = (hid_dim,) if isinstance(hid_dim, int) else tuple(default(hid_dim, ()))
        if any(w <= 0 or w % 64 for w in hid_dim + (d_out,)):
            raise NotImplementedError(f'SpaceTimeAttention: hid_dim {hid_dim} and d_out {d_out} must be positive '
                                      f'multiples of 64 (the channel blocks of the convolution GEMMs)')
        self.space_attn = SpatialAttention(n_head=n_head[0], d_head=d_head[0], bias=bias, scale=scale, embed=embed[0],
                                           causal=False, dropout=dropout, transpose=transpose, **space_attn_kw)
        self.temp_attn = TemporalAttention(n_head=n_head[1], d_head=d_head[1], bias=bias, scale=scale, embed=embed[1],
                                           causal=True, dropout=dropout, transpose=transpose, **time_attn_kw)
        # nn.Sequential(Rearrange, ForwardBlock, Rearrange): ForwardBlock sits at index 1 -> keys 'ffn.1.net...'
        self.ffn = nn.Sequential(nn.Identity(), _FfnNet(dim, d_out, hid_dim, n_head[1], kernel_size, bias),
                                 nn.Identity())
        self.in_channels, self.out_channels = dim, d_out
        self.transpose = transpose
        self.time_skip = nn.Identity()
        self.space_skip = nn.Identity()
        # nn.Conv3d(dim, d_out, 1) (bias on) in the reference; runs as extra K columns of the last FFN conv
        self.ffn_skip = Conv3dParams(dim, d_out, 1, causal=False) if d_out != dim else nn.Identity()
        self._fuse_skip()

    def _fuse_skip(self):
        if isinstance(self.ffn_skip, Conv3dParams):
            self.ffn[1].net[-1][0].fuse_shortcut(self.ffn_skip)

    def __setstate__(self, state):
        super().__setstate__(state)
        self._fuse_skip()     # re-link inside the copy (see Conv3dParams.__setstate__)

    def forward(self, video: Tensor, cond=None, mask: Tensor | None = None) -> Tensor:
        if not isinstance(cond, tuple):
            cond = (cond, cond)
        space_cond, time_cond = cond
        if exists(space_cond) and self.transpose is not None and not isinstance(space_cond, Tensor):
            space_cond = None
        if exists(mask):
            raise NotImplementedError('mask must stay None (SDPA forbids attn_mask with is_causal)')
        x = video.permute(0, 2, 3, 4, 1) if self.transpose else video
        x = self.space_attn(x, transpose=False, _residual=True)
        # LatentAction passes cond=(None, q_act); a bare tensor cond is the temporal one too
        tc = time_cond if isinstance(self.temp_attn.to_qkv.to_k, nn.Linear) else None
        x = self.temp_attn(x, cond=tc, transpose=False, _residual=True)
        gn = self.ffn[1].net[0]
        convs = [(c.weight, c.bias, c.packed(), c.geom) for c in (layer[0] for layer in self.ffn[1].net[1:])]
        skip = self.ffn_skip if isinstance(self.ffn_skip, Conv3dParams) else None
        x = ops.ffn_res(x, gn.weight, gn.bias, convs, gn.num_groups, gn.eps, *((skip.weight, skip.bias) if skip else ()))
        return x.permute(0, 4, 1, 2, 3) if self.transpose else x
