"""Blueprint registry — same names and semantics as genie/module/__init__.py:23-93.

Names the reference registers but no shipped blueprint uses ('causal-conv3d-transpose',
'depth2space_upsample', 'depth2time_upsample', the 2-D image modules) are outside the hot-path scope
(SURVEY.md §8) and raise NotImplementedError rather than silently running a PyTorch fallback."""
from typing import List, Tuple

import torch.nn as nn

from ..utils import Blueprint, default, exists
from .norm import AdaptiveGroupNorm, GroupNorm, SiLU
from .image import BlurPooling2d
from .video import CausalConv3d, DepthToSpaceTimeUpsample, SpaceTimeDownsample, VideoResidualBlock

_OUT_OF_SCOPE = ('space_downsample', 'image-residual', 'causal-conv3d-transpose',
                 'depth2space_upsample', 'depth2time_upsample', 'gelu', 'relu', 'leaky_relu')


def get_module(name: str):
    match name:
        case 'space_attn':
            from .attention import SpatialAttention
            return SpatialAttention
        case 'time_attn':
            from .attention import TemporalAttention
            return TemporalAttention
        case 'space-time_attn':
            from .attention import SpaceTimeAttention
            return SpaceTimeAttention
        case 'blur_pool':
            return BlurPooling2d
        case 'video-residual':
            return VideoResidualBlock
        case 'causal-conv3d':
            return CausalConv3d
        case 'depth2spacetime_upsample':
            return DepthToSpaceTimeUpsample
        case 'spacetime_downsample':
            return SpaceTimeDownsample
        case 'group_norm':
            return GroupNorm
        case 'adaptive_group_norm':
            return AdaptiveGroupNorm
        case 'silu':
            return SiLU
        case _ if name in _OUT_OF_SCOPE:
            raise NotImplementedError(f'module {name!r} is registered by the reference but lies outside the '
                                      f'hot-path scope (no shipped blueprint uses it)')
        case _:
            raise ValueError(f'Unknown module name: {name}')


def parse_blueprint(blueprint: Blueprint) -> Tuple[nn.ModuleList, List[bool]]:
    """Expand a blueprint into layers + per-layer `has_ext` flags (genie/module/__init__.py:71-93).
    Unlike the reference this does NOT mutate the caller's dicts (the reference pops 'n_rep'/'has_ext',
    so re-parsing the same blueprint object there silently builds a different network)."""
    layers, ext_kw = [], []
    for desc in blueprint:
        if isinstance(desc, str):
            desc = (desc, {})
        name, kwargs = default(desc, (None, {}))
        kwargs = dict(kwargs)
        has_ext = kwargs.pop('has_ext', False)
        n_rep = kwargs.pop('n_rep', 1)
        ext_kw.extend([has_ext] * n_rep)
        if exists(name):
            layers.extend(get_module(name)(**kwargs) for _ in range(n_rep))
    return nn.ModuleList(layers), ext_kw
