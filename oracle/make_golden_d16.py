"""oracle/make_golden_d16.py — tests/golden/attn_d16.pt by RUNNING THE REAL REFERENCE.   TEST INFRASTRUCTURE.

    OPEN_GENIE_REFERENCE=/path/to/open-genie python oracle/make_golden_d16.py

Attention heads of width 16, the width of every space-time blueprint the reference ships (LATENT_ACT_ENC / DEC, the
README's examples, its test_dynamics.py / test_action.py), run as oracle/make_golden.py runs its models: unmodified
reference modules, closed-form weights and inputs, CPU fp32. Every result is compared with oracle.genie_oracle (a
mismatch aborts). Cases:
  * SpaceTimeAttention(4, 16) with transpose False / True, frames of S = 64, 100 and 256 tokens, with and without
    temporal conditioning; SpaceTimeAttention(16, 16) at 256 channels; the mixed block n_head = (4, 1),
    d_head = (16, 64). Loss = mean(y^2).
  * DynamicsModel in the configuration of the reference's test/test_dynamics.py (without its n_embd key): 4 blocks of
    4 heads of 16 at embed_dim 64, tokens (2, 10, 16, 16) with an explicit mask. compute_loss and its gradients, and
    the forward logits.
  * LatentAction with the mini blueprints narrowed to 8 heads of 16, with quant.proj_inp / proj_out pinned to Identity
    as make_golden.py pins them. The training loss and its gradients.
Stored per case, to keep the file small: shapes, every gradient's norm, and samples at oracle.genie_oracle.det_indices
positions of the outputs, dx and each gradient.
"""
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG                    # noqa: E402  (puts the reference and this repository on sys.path)
from make_golden import DynamicsModel, LatentAction, SpaceTimeAttention  # noqa: E402  (the reference's)

from oracle import fixtures as fx           # noqa: E402
from oracle import genie_oracle as O        # noqa: E402

D = 16
# (tag, n_head, d_head, transpose, key_dim or None, input shape)
ST_CASES = (
    ('h4_t0_s64', 4, D, False, None, (2, 3, 8, 8, 64)),
    ('h4_t0_s100_c4', 4, D, False, 4, (2, 3, 10, 10, 64)),
    ('h4_t0_s256', 4, D, False, None, (1, 2, 16, 16, 64)),
    ('h4_t1_s64_c4', 4, D, True, 4, (2, 64, 3, 8, 8)),
    ('h4_t1_s100', 4, D, True, None, (2, 64, 3, 10, 10)),
    ('h4_t1_s256_c4', 4, D, True, 4, (1, 64, 2, 16, 16)),
    ('h16_t0_s64', 16, D, False, None, (2, 2, 8, 8, 256)),
    ('mixed_t0_s64', (4, 1), (D, 64), False, None, (2, 3, 8, 8, 64)),
)
DYN_DESC = (('space-time_attn', {'n_rep': 4, 'n_head': 4, 'd_head': D, 'transpose': False}),)
DYN = dict(tok_vocab=16, act_vocab=4, embed_dim=64)
DYN_TOKENS_SHAPE = (2, 10, 16, 16)
N_OUT, N_GRAD = 256, 32          # sampled elements of an output, and of each gradient


def narrow(bp):
    """A blueprint with every space-time block at 8 heads of 16 (the mini blueprints' 128 channels)."""
    return tuple((n, {**kw, 'n_head': 8, 'd_head': D} if n == 'space-time_attn' else kw) for n, kw in bp)


def sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)].clone()


def st_inputs(tag, transpose, cond_dim, shape):
    x = O.det_uniform(f'd16.x.{tag}', shape)
    t = shape[2] if transpose else shape[1]
    cond = O.det_uniform(f'd16.cond.{tag}', (shape[0], t, cond_dim)).sign() if cond_dim else None
    return x, cond


def st_oracle(sd, x, nh, transpose, cond):
    """oracle.genie_oracle's block; the mixed block composed from its parts (GroupNorm over the temporal head count)."""
    if isinstance(nh, int):
        return O.spacetime_attention(sd, '', x, nh, transpose, cond)
    x = x.movedim(1, -1) if transpose else x
    x = O.spatial_attention(sd, 'space_attn.', x, nh[0], False) + x
    x = O.temporal_attention(sd, 'temp_attn.', x, nh[1], False, cond) + x
    y = F.group_norm(x.movedim(-1, 1), nh[1], sd['ffn.1.net.0.weight'], sd['ffn.1.net.0.bias'], 1e-5)
    y = F.conv3d(y, sd['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x
    return y.movedim(-1, 1) if transpose else y


def grad_record(prefix, grads):
    names = sorted(grads)
    return {'grad_names': names, 'grad_norm': {k: grads[k].norm().item() for k in names},
            'grad': {k: sample(f'{prefix}.{k}', grads[k], N_GRAD) for k in names}}


def gen_blocks(out):
    for tag, nh, dh, transpose, cond_dim, shape in ST_CASES:
        kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
        m = SpaceTimeAttention(n_head=nh, d_head=dh, transpose=transpose, **kw)
        sd = MG.load_det(m)
        x, cond = st_inputs(tag, transpose, cond_dim, shape)
        x.requires_grad_(True)
        y = m(x, cond=(None, cond)) if cond_dim else m(x)
        y.square().mean().backward()
        grads = MG.grads_of(m)
        ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
        xo = x.detach().clone().requires_grad_(True)
        yo = st_oracle(ref, xo, nh, transpose, cond)
        yo.square().mean().backward()
        MG.close(yo, y, f'SpaceTimeAttention {tag}', rtol=2e-4, atol=2e-5)
        MG.close(xo.grad, x.grad, f'  dx {tag}', rtol=2e-4, atol=1e-6)
        for k, g in grads.items():
            MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
        out[tag] = {'n_head': nh, 'd_head': dh, 'transpose': transpose, 'key_dim': cond_dim, 'shape': shape,
                    'keys': {k: tuple(v.shape) for k, v in sd.items()}, 'y': sample(f'd16.y.{tag}', y, N_OUT),
                    'dx': sample(f'd16.dx.{tag}', x.grad, N_OUT), **grad_record(f'd16.g.{tag}', grads)}


def gen_dynamics(out):
    dm = DynamicsModel(desc=fx.bp(DYN_DESC), **DYN)
    sd = MG.load_det(dm)
    u = O.det_uniform('d16.dyn.tokens', DYN_TOKENS_SHAPE) / (3 ** 0.5)            # in (-1, 1)
    tokens = ((u + 1) * 0.5 * DYN['tok_vocab']).long().clamp(0, DYN['tok_vocab'] - 1)
    ua = O.det_uniform('d16.dyn.act', DYN_TOKENS_SHAPE[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * DYN['act_vocab']).long().clamp(0, DYN['act_vocab'] - 1)
    mask = O.det_uniform('d16.dyn.mask', DYN_TOKENS_SHAPE) / (3 ** 0.5) < 0.5     # ~75 % masked
    logits, _ = dm(tokens, act)
    MG.close(O.dynamics_forward(sd, DYN_DESC, tokens, act), logits, 'Dynamics logits', rtol=2e-4, atol=2e-5)
    loss = dm.compute_loss(tokens, act, mask=mask)
    loss.backward()
    grads = MG.grads_of(dm)
    ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
    oloss = O.dynamics_loss(ref, DYN_DESC, tokens, act, mask)
    oloss.backward()
    MG.close(oloss, loss, 'Dynamics loss', rtol=2e-4)
    for k, g in grads.items():
        MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
    out['dynamics'] = {'desc': DYN_DESC, 'kw': DYN, 'tokens': tokens, 'act': act, 'mask': mask,
                       'keys': {k: tuple(v.shape) for k, v in sd.items()}, 'logits_shape': tuple(logits.shape),
                       'logits': sample('d16.dyn.logits', logits, N_OUT), 'loss': loss.item(),
                       **grad_record('d16.dyn.g', grads)}


def gen_latent_action(out):
    enc, dec = narrow(fx.MINI_ACT_ENC), narrow(fx.MINI_ACT_DEC)
    la = LatentAction(fx.bp(enc), fx.bp(dec), d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                      inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    la.quant.proj_inp = la.quant.proj_out = nn.Identity()      # constructor omits input_dim (action.py:93-101)
    sd = MG.load_det(la)
    video = O.det_uniform('d16.action.video', fx.MINI_ACT_VIDEO_SHAPE)
    la.train()
    idxs, loss, (rec_loss, q_loss) = la(video)
    loss.backward()
    oidx, oloss, (orec, _), _ = O.latent_action_forward(sd, enc, dec, video, fx.MINI_ACT_D_CODEBOOK)
    MG.close(oidx, idxs, 'LatentAction idxs')
    MG.close(oloss, loss, 'LatentAction loss', rtol=2e-4)
    MG.close(orec, rec_loss, 'LatentAction rec loss', rtol=2e-4)
    out['latent_action'] = {'enc': enc, 'dec': dec, 'idxs': idxs, 'loss': loss.item(), 'rec_loss': rec_loss.item(),
                            'q_loss': q_loss.item(), **grad_record('d16.action.g', MG.grads_of(la))}


def main():
    out = {}
    gen_blocks(out)
    gen_dynamics(out)
    gen_latent_action(out)
    path = os.path.join(MG.OUT, 'attn_d16.pt')
    torch.save(out, path)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
