"""oracle/causal_oracle.py — causal and grouped video residual blocks, restated in plain torch.   TEST INFRASTRUCTURE.

Extends oracle.genie_oracle (which restates the MAGVIT2 blocks: use_causal=False, SiLU) to every option of
VideoResidualBlock the CUDA modules implement, and to the models built from them:
  * video_residual_block: use_causal (CausalConv3d pads and 'conv3d' keys), the activation, num_groups in the
    GroupNorms and in the blur pooling of `downsample` (genie/module/video.py:539-656, 487-537, 106-200);
  * video_discriminator: VideoDiscriminator without attention (genie/module/discriminator.py:116-221);
  * run_layers / tokenizer_forward / tokenizer_tokenize: the tokenizer's layer loop with these blocks;
  * CAUSAL_ENC / CAUSAL_DEC: this project's causal mini tokenizer blueprint.
oracle/make_golden_causal.py checks every function here against the unmodified reference.
"""
import torch.nn.functional as F
from torch import Tensor

from oracle import genie_oracle as O

# A causal mini tokenizer shaped like a MAGVIT-v2 causal encoder: causal stem, a causal block that halves space
# through blur pooling, a plain block that widens, a causal grouped block that halves time and space, and a
# GroupNorm / SiLU / 1x1x1 head into the LFQ. The decoder mirrors it with causal blocks on the fused path (no
# down-sampling), one of them grouped. Video (2, 3, 8, 32, 32) -> latent (2, 6, 4, 8, 8).
CAUSAL_ENC = (
    ('causal-conv3d', {'in_channels': 3, 'out_channels': 64, 'kernel_size': 3}),
    ('video-residual', {'in_channels': 64, 'kernel_size': 3, 'downsample': (1, 2), 'use_causal': True}),
    ('video-residual', {'in_channels': 64, 'out_channels': 128}),
    ('video-residual', {'in_channels': 128, 'kernel_size': 3, 'downsample': 2, 'use_causal': True, 'num_groups': 2}),
    ('group_norm', {'num_groups': 8, 'num_channels': 128}),
    ('silu', {}),
    ('causal-conv3d', {'in_channels': 128, 'out_channels': 6, 'kernel_size': 1}),
)
CAUSAL_DEC = (
    ('causal-conv3d', {'in_channels': 6, 'out_channels': 128, 'kernel_size': 3}),
    ('video-residual', {'in_channels': 128, 'use_causal': True}),
    ('depth2spacetime_upsample', {'in_channels': 128, 'kernel_size': 3, 'time_factor': 2, 'space_factor': 2}),
    ('video-residual', {'in_channels': 128, 'out_channels': 64, 'use_causal': True, 'num_groups': 2}),
    ('depth2spacetime_upsample', {'in_channels': 64, 'kernel_size': 3, 'time_factor': 1, 'space_factor': 2}),
    ('video-residual', {'in_channels': 64}),
    ('group_norm', {'num_groups': 8, 'num_channels': 64}),
    ('silu', {}),
    ('causal-conv3d', {'in_channels': 64, 'out_channels': 3, 'kernel_size': 3}),
)
CAUSAL_D_CODEBOOK = 6
CAUSAL_VIDEO_SHAPE = (2, 3, 8, 32, 32)

ACT = {'swish': F.silu, 'silu': F.silu, 'leaky': F.leaky_relu, 'relu': F.relu}


def video_residual_block(sd, pre: str, x: Tensor, num_groups: int = 1, downsample=None, use_causal: bool = False,
                         act_fn: str = 'swish') -> Tensor:
    """VideoResidualBlock.forward — video.py:578-631 (layers) and 648 (main(x) + res(x)).

    main = GN -> act -> conv(k) -> [blur] -> GN -> act -> conv(k); res = [blur] -> conv(1x1x1). A causal block's convs
    pad time by kt - 1 in front and space by (k - 1) // 2 (CausalConv3d); a plain block's pad every dimension by
    (k - 1) // 2. The blur pooling pads time symmetrically in both. `downsample` is an int or (time, space)."""
    act = ACT[act_fn]
    if isinstance(downsample, int):
        downsample = (downsample, downsample)

    def conv(h, name):
        if use_causal:
            return O.causal_conv3d(h, sd[pre + name + '.conv3d.weight'], sd[pre + name + '.conv3d.bias'])
        w = sd[pre + name + '.weight']
        return F.conv3d(h, w, sd[pre + name + '.bias'], padding=tuple((k - 1) // 2 for k in w.shape[2:]))

    k = sd[pre + ('main.2.conv3d.weight' if use_causal else 'main.2.weight')].shape[2]
    h = act(F.group_norm(x, num_groups, sd[pre + 'main.0.weight'], sd[pre + 'main.0.bias'], 1e-5))
    h = conv(h, 'main.2')
    if downsample is not None:
        h = O.blur_pool3d(h, k, downsample[0], downsample[1], num_groups)
        x = O.blur_pool3d(x, k, downsample[0], downsample[1], num_groups)
    h = act(F.group_norm(h, num_groups, sd[pre + 'main.4.weight'], sd[pre + 'main.4.bias'], 1e-5))
    return conv(h, 'main.6') + conv(x, 'res.1')


def video_discriminator(sd, video: Tensor, dims, down_step, num_groups: int = 1, act_fn: str = 'leaky') -> Tensor:
    """VideoDiscriminator.forward without attention — discriminator.py:139-221: Conv3d(k3, p1) stem, residual blocks
    each followed by the Identity attention and feed-forward residuals (x -> 4x), Conv3d(k3, p1) -> LeakyReLU ->
    flatten -> Linear. `dims` are the channel counts model_dim * dim_mults."""
    x = F.conv3d(video, sd['proj_in.weight'], sd['proj_in.bias'], padding=1)
    for i, down in enumerate(down_step[:len(dims) - 1]):        # zip(pairwise(dims), down_step)
        x = video_residual_block(sd, f'core.{i}.0.', x, num_groups, down, act_fn=act_fn)
        x = 4 * x
    x = F.leaky_relu(F.conv3d(x, sd['to_logits.0.weight'], sd['to_logits.0.bias'], padding=1))
    return F.linear(x.flatten(1), sd['to_logits.3.weight'], sd['to_logits.3.bias'])[:, 0]


def run_layers(sd, prefix: str, bp, x: Tensor) -> Tensor:
    """oracle.genie_oracle.run_layers with every VideoResidualBlock option."""
    for i, (name, kw) in enumerate(O.expand_blueprint(bp)):
        pre = f'{prefix}.{i}.'
        if name == 'video-residual':
            x = video_residual_block(sd, pre, x, kw.get('num_groups', 1), kw.get('downsample'),
                                     kw.get('use_causal', False), kw.get('act_fn', 'swish'))
        else:
            x = _one_layer(sd, pre, name, kw, x)
    return x


def _one_layer(sd, pre, name, kw, x):
    if name == 'causal-conv3d':
        return O.causal_conv3d(x, sd[pre + 'conv3d.weight'], sd.get(pre + 'conv3d.bias'))
    if name == 'depth2spacetime_upsample':
        return O.depth2spacetime_upsample(sd, pre, x, kw.get('time_factor', 2), kw.get('space_factor', 2))
    if name == 'spacetime_downsample':
        return O.spacetime_downsample(sd, pre, x, kw.get('time_factor', 2), kw.get('space_factor', 2))
    if name == 'group_norm':
        return F.group_norm(x, kw['num_groups'], sd[pre + 'weight'], sd[pre + 'bias'], 1e-5)
    if name == 'silu':
        return F.silu(x)
    raise ValueError(f'causal oracle: module {name!r} is not used by the causal blueprints')


def tokenizer_tokenize(sd, enc_bp, video: Tensor, d_codebook: int, beta: float = 100.):
    """VideoTokenizer.tokenize — tokenizer.py:332-350 (eval-mode LFQ)."""
    enc = run_layers(sd, 'enc_layers', enc_bp, video)
    (q, idxs), _ = O.lfq(enc, d_codebook, training=False, beta=beta, transpose=True,
                         proj_inp=O._lfq_proj(sd, 'proj_inp'), proj_out=O._lfq_proj(sd, 'proj_out'))
    return q, idxs


def tokenizer_forward(sd, enc_bp, dec_bp, video: Tensor, d_codebook: int, beta: float = 100.):
    """VideoTokenizer.forward in training mode with the GAN / perceptual terms at zero weight — tokenizer.py:352-387.
    Returns (loss, (rec_loss, quant_loss), rec_video, idxs)."""
    enc = run_layers(sd, 'enc_layers', enc_bp, video)
    (q, idxs), q_loss = O.lfq(enc, d_codebook, training=True, beta=beta, transpose=True,
                              proj_inp=O._lfq_proj(sd, 'proj_inp'), proj_out=O._lfq_proj(sd, 'proj_out'))
    rec = run_layers(sd, 'dec_layers', dec_bp, q)
    rec_loss = F.mse_loss(rec, video)
    return rec_loss + q_loss, (rec_loss, q_loss), rec, idxs
