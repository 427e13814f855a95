"""oracle/ffn_oracle.py — CPU restatement of SpaceTimeAttention with the reference's full feed-forward block.
*** TEST INFRASTRUCTURE ***

`oracle.genie_oracle.spacetime_attention` restates the block in its default form (GroupNorm -> one k = 3 conv, no bias,
+ x). This module restates every form the reference builds (genie/module/attention.py:373-474, ForwardBlock in
genie/module/misc.py:71-104) and reads the form from the state-dict keys:
    ffn.1.net.{i}.0.weight (and .bias)  i = 1 .. n   the convs, kernel size from the weight, padding (k-1)//2;
                                                     nn.GELU() (exact erf) after every conv but the last
    ffn_skip.{weight,bias}                           the 1x1x1 skip conv when d_out != n_head*d_head (transpose=True)
    temp_attn.to_qkv.to_{k,v}.bias                   the conditioning projections' biases (bias=True with key_dim)
It is pinned against the running reference by oracle/make_golden_ffn.py. `blueprints()` swaps it into
oracle.genie_oracle for the blueprint-level restatements (run_layers, dynamics_loss, latent_action_forward).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import genie_oracle as O

_default_block = O.spacetime_attention


def _cond_with_bias(sd, pre: str, cond: Tensor):
    """F.linear(c, W, b) == F.linear([c, 1], [W | b]): the restatement's attention core takes Linear weights only, so a
    bias rides along as one more input column of the condition."""
    kb, vb = sd.get(pre + 'to_qkv.to_k.bias'), sd.get(pre + 'to_qkv.to_v.bias')
    if kb is None and vb is None:
        return sd, cond
    sd = dict(sd)
    ones = torch.ones(cond.shape[:-1] + (1,), dtype=cond.dtype)
    for name, b in (('to_k', kb), ('to_v', vb)):
        w = sd[pre + f'to_qkv.{name}.weight']
        sd[pre + f'to_qkv.{name}.weight'] = torch.cat([w, (torch.zeros_like(w[:, :1]) if b is None else b[:, None])], 1)
    return sd, torch.cat([cond, ones], -1)


def ffn(sd, pre: str, x: Tensor, n_head: int) -> Tensor:
    """ffn(x) + ffn_skip(x) on a (b, c, t, h, w) tensor — attention.py:429-454, 472."""
    y = F.group_norm(x, n_head, sd[pre + 'ffn.1.net.0.weight'], sd[pre + 'ffn.1.net.0.bias'], 1e-5)
    n = 1
    while pre + f'ffn.1.net.{n + 1}.0.weight' in sd:
        n += 1
    for i in range(1, n + 1):
        w = sd[pre + f'ffn.1.net.{i}.0.weight']
        y = F.conv3d(y, w, sd.get(pre + f'ffn.1.net.{i}.0.bias'), padding=(w.shape[-1] - 1) // 2)
        if i < n:
            y = F.gelu(y)
    if pre + 'ffn_skip.weight' in sd:
        x = F.conv3d(x, sd[pre + 'ffn_skip.weight'], sd[pre + 'ffn_skip.bias'])
    return y + x


def spacetime_attention(sd, pre: str, video: Tensor, n_head: int, transpose: bool,
                        time_cond: Tensor | None = None) -> Tensor:
    """SpaceTimeAttention.forward — attention.py:456-474 with d_inp unset (space_skip, time_skip Identity)."""
    x = O.spatial_attention(sd, pre + 'space_attn.', video, n_head, transpose) + video
    if time_cond is not None:
        tsd, tc = _cond_with_bias(sd, pre + 'temp_attn.', time_cond)
    else:
        tsd, tc = sd, None
    x = O.temporal_attention(tsd, pre + 'temp_attn.', x, n_head, transpose, tc) + x
    y = ffn(sd, pre, x if transpose else x.movedim(-1, 1), n_head)   # Rearrange -> b c t h w
    return y if transpose else y.movedim(1, -1)


@contextlib.contextmanager
def blueprints():
    """Within the block, oracle.genie_oracle's blueprint restatements run every space-time block through
    spacetime_attention above."""
    O.spacetime_attention = spacetime_attention
    try:
        yield
    finally:
        O.spacetime_attention = _default_block
