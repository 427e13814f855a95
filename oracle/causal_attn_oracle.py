"""Spatial and temporal attention with SDPA's `is_causal` as a parameter (attention.py:196, 229-234): the reference's
SpatialAttention(causal=True) and TemporalAttention(causal=False), which genie_oracle.spatial_attention /
temporal_attention (fixed to the SpaceTimeAttention choices, False and True) do not cover. Both are those functions
with the flag passed through to genie_oracle.attention_core. TEST INFRASTRUCTURE."""
from __future__ import annotations

from torch import Tensor

from oracle import genie_oracle as O


def spatial_attention(sd, pre: str, video: Tensor, n_head: int, transpose: bool, causal: bool) -> Tensor:
    """SpatialAttention.forward (attention.py:279-307): SDPA over the h*w tokens of each frame in raster order."""
    x = video.movedim(1, -1) if transpose else video               # -> b t h w c
    b, t, h, w, c = x.shape
    o = O.attention_core(sd, pre, x.reshape(b * t, h * w, c), n_head, causal, '2d')
    o = o.reshape(b, t, h, w, c)
    return o.movedim(-1, 1) if transpose else o


def temporal_attention(sd, pre: str, video: Tensor, n_head: int, transpose: bool, causal: bool,
                       cond: Tensor | None = None) -> Tensor:
    """TemporalAttention.forward (attention.py:347-371): SDPA over t for every pixel; cond (b, t, k) repeated over
    (h, w)."""
    x = video.movedim(1, -1) if transpose else video               # b t h w c
    b, t, h, w, c = x.shape
    x = x.permute(0, 2, 3, 1, 4).reshape(b * h * w, t, c)
    if cond is not None:
        cond = cond[:, None, None].expand(b, h, w, *cond.shape[1:]).reshape(b * h * w, *cond.shape[1:])
    o = O.attention_core(sd, pre, x, n_head, causal, '1d', cond)
    o = o.reshape(b, h, w, t, c).permute(0, 3, 1, 2, 4)
    return o.movedim(-1, 1) if transpose else o
