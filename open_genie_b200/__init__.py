"""open_genie_b200 — H100-native (sm_90a) implementation of open-genie's data-parallel hot path behind the
reference's own Python surface (myscience/open-genie: genie/__init__.py).

Importing this package never touches the GPU; the CUDA library (csrc/libopengenie_b200.so) is loaded on
first use and there is no CPU or PyTorch fallback behind it."""
from .tokenizer import MAGVIT2_DEC_DESC, MAGVIT2_ENC_DESC, REPR_TOK_DEC, REPR_TOK_ENC, VideoTokenizer
from .action import LatentAction
from .dynamics import DynamicsModel
from .genie import Genie
from .module import get_module, parse_blueprint
from .optim import FusedAdamW
from .ops import enable_zero_arena
from .data import LightningDataset, LightningPlatformer2D, Platformer2D, VideoBatchPrefetcher, frames_to_video

# LATENT_ACT_* blueprints: the intent of genie/__init__.py:10-54 in its HEAD-valid form (SURVEY.md §8): `n_embd`
# dropped (SpaceTimeAttention does not accept it), heads 4 x 64 = 256 = n_embd, 'spacetime_upsample' (not in the
# registry) -> 'depth2spacetime_upsample'.
LATENT_ACT_ENC = (
    ('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 64, 'transpose': True}),
    ('spacetime_downsample', {'in_channels': 256, 'kernel_size': 3, 'time_factor': 1, 'space_factor': 2}),
    ('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 64, 'transpose': True}),
)
LATENT_ACT_DEC = (
    ('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 64, 'transpose': True, 'has_ext': True,
                         'time_attn_kw': {'key_dim': 8}}),
    ('depth2spacetime_upsample', {'in_channels': 256, 'kernel_size': 3, 'time_factor': 1, 'space_factor': 2}),
    ('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 64, 'transpose': True, 'has_ext': True,
                         'time_attn_kw': {'key_dim': 8}}),
)

__all__ = ['VideoTokenizer', 'LatentAction', 'DynamicsModel', 'Genie', 'LATENT_ACT_ENC', 'LATENT_ACT_DEC', 'MAGVIT2_ENC_DESC', 'MAGVIT2_DEC_DESC', 'REPR_TOK_ENC', 'REPR_TOK_DEC',
           'get_module', 'parse_blueprint', 'FusedAdamW', 'enable_zero_arena', 'LightningDataset', 'LightningPlatformer2D', 'Platformer2D',
           'VideoBatchPrefetcher', 'frames_to_video']
