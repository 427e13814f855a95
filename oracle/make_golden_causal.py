"""oracle/make_golden_causal.py — tests/golden/causal_resblock.pt by RUNNING THE REAL REFERENCE.   TEST INFRASTRUCTURE.

    OPEN_GENIE_REFERENCE=/path/to/open-genie python oracle/make_golden_causal.py

Causal and grouped video residual blocks, run as oracle/make_golden.py runs its models: unmodified reference modules,
closed-form weights and inputs, CPU fp32. Every output and gradient is compared with oracle.causal_oracle (a mismatch
aborts). Cases:
  * the four VideoResidualBlock configurations of the reference's test/test_video.py (64 -> 128 on (1, 64, 8, 16, 16):
    plain; causal with num_groups = 2; LeakyReLU with downsample (2, 4); all of these together);
  * causal blocks 128 -> 256 with downsample (1, 2) and 2, and a causal block at kernel_size 1;
  * BlurPooling3d alone with num_groups = 4 and 64 -> 128 channels, on ragged extents;
  * VideoDiscriminator(num_groups = 2);
  * the causal mini tokenizer of oracle.causal_oracle: tokenize, decode, and the training loss with its gradients.
Block and pooling losses are mean(y^2). Stored per case, to keep the file small: shapes, every gradient's norm, and
samples at oracle.genie_oracle.det_indices positions of the outputs, dx and each gradient.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG                    # noqa: E402  (puts the reference and this repository on sys.path)
from make_golden import BlurPooling3d, VideoResidualBlock, VideoTokenizer  # noqa: E402  (the reference's)

from oracle import causal_oracle as C       # noqa: E402
from oracle import genie_oracle as O        # noqa: E402

# (tag, VideoResidualBlock kwargs, input shape)
BLOCK_CASES = (
    ('video_plain', dict(in_channels=64, out_channels=128), (1, 64, 8, 16, 16)),
    ('video_causal_g2', dict(in_channels=64, out_channels=128, num_groups=2, use_causal=True), (1, 64, 8, 16, 16)),
    ('video_leaky_down24', dict(in_channels=64, out_channels=128, downsample=(2, 4), act_fn='leaky'),
     (1, 64, 8, 16, 16)),
    ('video_causal_g2_leaky_down24', dict(in_channels=64, out_channels=128, num_groups=2, use_causal=True,
                                          act_fn='leaky', downsample=(2, 4)), (1, 64, 8, 16, 16)),
    ('causal_down12', dict(in_channels=128, out_channels=256, downsample=(1, 2), use_causal=True), (2, 128, 4, 8, 8)),
    ('causal_down2', dict(in_channels=128, out_channels=256, downsample=2, use_causal=True), (2, 128, 4, 8, 8)),
    ('causal_k1', dict(in_channels=64, out_channels=128, kernel_size=1, use_causal=True), (2, 64, 4, 8, 8)),
)
BLUR_CASE = dict(in_channels=64, kernel_size=3, out_channels=128, time_factor=2, space_factor=2, num_groups=4)
BLUR_SHAPE = (2, 64, 5, 9, 11)
DISC_KW = dict(inp_size=(8, 16, 16), num_groups=2)
DISC_SHAPE = (2, 3, 8, 16, 16)
N_OUT, N_GRAD = 256, 32          # sampled elements of an output, and of each gradient


def sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)].clone()


def grad_record(prefix, grads):
    names = sorted(grads)
    return {'grad_names': names, 'grad_norm': {k: grads[k].norm().item() for k in names},
            'grad': {k: sample(f'{prefix}.{k}', grads[k], N_GRAD) for k in names}}


def run_case(tag, m, shape, oracle):
    """mean(y^2) through the reference module `m` and through `oracle(sd, x)`; both must agree."""
    sd = MG.load_det(m)
    x = O.det_uniform(f'causal.x.{tag}', shape).requires_grad_(True)
    y = m(x)
    y.square().mean().backward()
    grads = MG.grads_of(m)
    ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
    xo = x.detach().clone().requires_grad_(True)
    yo = oracle(ref, xo)
    yo.square().mean().backward()
    MG.close(yo, y, tag, rtol=2e-4, atol=2e-5)
    MG.close(xo.grad, x.grad, f'  dx {tag}', rtol=2e-4, atol=1e-6)
    for k, g in grads.items():
        MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
    return {'shape': shape, 'keys': {k: tuple(v.shape) for k, v in sd.items()}, 'y_shape': tuple(y.shape),
            'y': sample(f'causal.y.{tag}', y, N_OUT), 'dx': sample(f'causal.dx.{tag}', x.grad, N_OUT),
            **grad_record(f'causal.g.{tag}', grads)}


def gen_blocks(out):
    for tag, kw, shape in BLOCK_CASES:
        m = VideoResidualBlock(**kw)
        oracle = lambda sd, x, kw=kw: C.video_residual_block(
            sd, '', x, kw.get('num_groups', 1), kw.get('downsample'), kw.get('use_causal', False),
            kw.get('act_fn', 'swish'))
        out[tag] = {'kw': kw, **run_case(tag, m, shape, oracle)}
    m = BlurPooling3d(**BLUR_CASE)
    oracle = lambda sd, x: O.blur_pool3d(x, 3, 2, 2, BLUR_CASE['num_groups'], BLUR_CASE['out_channels'])
    out['blur_g4'] = {'kw': BLUR_CASE, **run_case('blur_g4', m, BLUR_SHAPE, oracle)}


def gen_discriminator(out):
    from genie.module.discriminator import VideoDiscriminator
    m = VideoDiscriminator(**DISC_KW)
    dims = [64 * k for k in (1, 2, 4)]
    oracle = lambda sd, x: C.video_discriminator(sd, x, dims, (None, 2, 2), DISC_KW['num_groups'])
    out['video_disc_g2'] = {'kw': DISC_KW, **run_case('video_disc_g2', m, DISC_SHAPE, oracle)}


def gen_tokenizer(out):
    enc, dec = C.CAUSAL_ENC, C.CAUSAL_DEC
    tok = VideoTokenizer(MG.fx.bp(enc), MG.fx.bp(dec), d_codebook=C.CAUSAL_D_CODEBOOK, gan_loss_weight=0,
                         perc_loss_weight=0)
    tok.gan_crit = tok.perc_crit = MG.ZeroLoss()
    sd = MG.load_det(tok)
    video = O.det_uniform('causal.tokenizer.video', C.CAUSAL_VIDEO_SHAPE)
    quant, idxs = tok.tokenize(video)
    oq, oidx = C.tokenizer_tokenize(sd, enc, video, C.CAUSAL_D_CODEBOOK)
    MG.close(oq, quant, 'tokenize quant')
    MG.close(oidx, idxs, 'tokenize idxs')
    enc_v = tok.encode(video).detach()
    dec_v = tok.decode(quant).detach()
    MG.close(C.run_layers(sd, 'dec_layers', dec, quant), dec_v, 'decode', rtol=2e-4, atol=2e-5)
    tok.train()
    loss, (rec_loss, _, _, _, q_loss) = tok(video)
    loss.backward()
    grads = MG.grads_of(tok)
    ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
    oloss, (orec, oq_loss), _, _ = C.tokenizer_forward(ref, enc, dec, video, C.CAUSAL_D_CODEBOOK)
    oloss.backward()
    MG.close(oloss, loss, 'tokenizer loss')
    MG.close(orec, rec_loss, 'rec loss')
    MG.close(oq_loss, q_loss, 'quant loss')
    for k, g in grads.items():
        MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-3, atol=1e-6)
    out['tokenizer'] = {'enc': enc, 'dec': dec, 'd_codebook': C.CAUSAL_D_CODEBOOK, 'video_shape': C.CAUSAL_VIDEO_SHAPE,
                        'keys': {k: tuple(v.shape) for k, v in sd.items()}, 'quant_shape': tuple(quant.shape),
                        'quant': sample('causal.tok.quant', quant, N_OUT), 'idxs': idxs.clone(),
                        'enc_shape': tuple(enc_v.shape), 'enc_latent': enc_v.clone(),
                        'decode_shape': tuple(dec_v.shape), 'decode': sample('causal.tok.decode', dec_v, N_OUT),
                        'loss': loss.item(), 'rec_loss': rec_loss.item(), 'quant_loss': q_loss.item(),
                        **grad_record('causal.tok.g', grads)}


def main():
    out = {}
    gen_blocks(out)
    gen_discriminator(out)
    gen_tokenizer(out)
    path = os.path.join(MG.OUT, 'causal_resblock.pt')
    torch.save(out, path)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
