"""oracle/noembed_oracle.py — attention without a rotary embedding (embed=False) in the CPU oracle.   TEST INFRASTRUCTURE.

With embed=False the reference replaces RotaryEmbedding by nn.Identity (genie/module/attention.py:199-239, 255-275,
323-343): q = k = v = LayerNorm(x), and the state_dict has no `embed.freq` entry for that attention. oracle.genie_oracle's
attention functions read `embed.freq`; a rotation by zero frequencies is the identity exactly in fp32
(x * cos 0 + rot(x) * sin 0 = x * 1 + rot(x) * 0 = x, and its gradient is the incoming one unchanged), so the oracle
of an embed=False module is genie_oracle run on its state_dict with zero frequencies supplied for every attention that
has none. oracle/make_golden_noembed.py checks this against the unmodified reference.
"""
from __future__ import annotations

from typing import Dict

import torch
from torch import Tensor

_ATTN_NORM = ('space_attn.norm.weight', 'temp_attn.norm.weight')


def identity_embed(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """A copy of the state_dict `sd` (shallow: the tensors are shared) with `embed.freq` = zeros(C / 2) added for every
    spatial or temporal attention that has no rotary embedding (a stand-alone attention's keys have no prefix)."""
    out = dict(sd)
    for k, w in sd.items():
        if k.endswith(_ATTN_NORM) or k == 'norm.weight':
            pre = k[:-len('norm.weight')]
            if pre + 'embed.freq' not in sd:
                out[pre + 'embed.freq'] = torch.zeros(w.shape[0] // 2, dtype=torch.float32)
    return out
