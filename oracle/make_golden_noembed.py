"""oracle/make_golden_noembed.py — tests/golden/attn_noembed.pt by RUNNING THE REAL REFERENCE.   TEST INFRASTRUCTURE.

    OPEN_GENIE_REFERENCE=/path/to/open-genie python oracle/make_golden_noembed.py

Attention without a rotary embedding (embed=False, where the reference's embedding is nn.Identity), run as
oracle/make_golden.py runs its models: unmodified reference modules, closed-form weights and inputs, CPU fp32. Every
result is compared with oracle.genie_oracle on the state_dict completed by oracle.noembed_oracle.identity_embed (a
mismatch aborts). Cases:
  * SpatialAttention(4, 16, embed=False) and TemporalAttention(4, 16, embed=False, causal=True) (as SpaceTimeAttention
    builds it), the latter also with a key_dim = 4 conditioning. The modules' outputs (no skip); loss = mean(y^2).
  * SpaceTimeAttention with embed False, (False, True) and (True, False) at d_head 16 (4 heads) and 64 (2 heads), one
    with temporal conditioning (key_dim = 4), one transposed, and the mixed block n_head = (4, 1), d_head = (16, 64).
    Loss = mean(y^2).
  * A DynamicsModel whose blueprint passes embed=False: compute_loss and its gradients, and the forward logits.
Stored per case: the configuration, the reference's state_dict keys and shapes, every gradient's norm, and samples at
oracle.genie_oracle.det_indices positions of the outputs, dx and each gradient.
"""
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG                    # noqa: E402  (puts the reference and this repository on sys.path)
from make_golden import DynamicsModel, SpaceTimeAttention  # noqa: E402  (the reference's)
from genie.module.attention import SpatialAttention, TemporalAttention  # noqa: E402  (the reference's)

from oracle import fixtures as fx           # noqa: E402
from oracle import genie_oracle as O        # noqa: E402
from oracle.noembed_oracle import identity_embed  # noqa: E402

# (tag, class name, n_head, d_head, key_dim or None, input shape (B, T, H, W, C))
ATTN_CASES = (
    ('spatial', 'SpatialAttention', 4, 16, None, (2, 3, 8, 8, 64)),
    ('temporal', 'TemporalAttention', 4, 16, None, (2, 12, 4, 4, 64)),
    ('temporal_c4', 'TemporalAttention', 4, 16, 4, (2, 12, 4, 4, 64)),
)
# (tag, n_head, d_head, embed, transpose, key_dim or None, input shape)
ST_CASES = (
    ('d16_e00', 4, 16, False, False, None, (2, 5, 8, 8, 64)),
    ('d16_e01', 4, 16, (False, True), False, None, (2, 5, 8, 8, 64)),
    ('d16_e10', 4, 16, (True, False), False, None, (2, 5, 8, 8, 64)),
    ('d16_e00_c4', 4, 16, False, False, 4, (2, 5, 8, 8, 64)),
    ('d16_e00_t1', 4, 16, False, True, None, (2, 64, 5, 8, 8)),
    ('d64_e00', 2, 64, False, False, None, (2, 5, 8, 8, 128)),
    ('d64_e01', 2, 64, (False, True), False, None, (2, 5, 8, 8, 128)),
    ('d64_e10', 2, 64, (True, False), False, None, (2, 5, 8, 8, 128)),
    ('mixed_e01', (4, 1), (16, 64), (False, True), False, None, (2, 5, 8, 8, 64)),
)
DYN_DESC = (('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 16, 'transpose': False, 'embed': False}),)
DYN = dict(tok_vocab=16, act_vocab=4, embed_dim=64)
DYN_TOKENS_SHAPE = (2, 6, 8, 8)
N_OUT, N_GRAD = 256, 32          # sampled elements of an output, and of each gradient


def sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)].clone()


def grad_record(prefix, grads):
    names = sorted(grads)
    return {'grad_names': names, 'grad_norm': {k: grads[k].norm().item() for k in names},
            'grad': {k: sample(f'{prefix}.{k}', grads[k], N_GRAD) for k in names}}


def inputs(tag, shape, t_axis, cond_dim):
    x = O.det_uniform(f'noembed.x.{tag}', shape)
    cond = O.det_uniform(f'noembed.cond.{tag}', (shape[0], shape[t_axis], cond_dim)).sign() if cond_dim else None
    return x, cond


def attn_oracle(sd, kind, x, nh, cond):
    sd = identity_embed(sd)
    if kind == 'SpatialAttention':
        return O.spatial_attention(sd, '', x, nh, False)
    return O.temporal_attention(sd, '', x, nh, False, cond)


def st_oracle(sd, x, nh, transpose, cond):
    """oracle.genie_oracle's block; the mixed block composed from its parts (GroupNorm over the temporal head count)."""
    sd = identity_embed(sd)
    if isinstance(nh, int):
        return O.spacetime_attention(sd, '', x, nh, transpose, cond)
    x = x.movedim(1, -1) if transpose else x
    x = O.spatial_attention(sd, 'space_attn.', x, nh[0], False) + x
    x = O.temporal_attention(sd, 'temp_attn.', x, nh[1], False, cond) + x
    y = F.group_norm(x.movedim(-1, 1), nh[1], sd['ffn.1.net.0.weight'], sd['ffn.1.net.0.bias'], 1e-5)
    y = F.conv3d(y, sd['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x
    return y.movedim(-1, 1) if transpose else y


def check_case(m, sd, y, x, oracle_fn, tag):
    """Backward of mean(y^2) through the reference and the oracle; every output and gradient compared."""
    y.square().mean().backward()
    grads = MG.grads_of(m)
    ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
    xo = x.detach().clone().requires_grad_(True)
    yo = oracle_fn(ref, xo)
    yo.square().mean().backward()
    MG.close(yo, y, tag, rtol=2e-4, atol=2e-5)
    MG.close(xo.grad, x.grad, f'  dx {tag}', rtol=2e-4, atol=1e-6)
    for k, g in grads.items():
        MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
    return {'keys': {k: tuple(v.shape) for k, v in sd.items()}, 'y': sample(f'noembed.y.{tag}', y, N_OUT),
            'dx': sample(f'noembed.dx.{tag}', x.grad, N_OUT), **grad_record(f'noembed.g.{tag}', grads)}


def gen_attention(out):
    for tag, kind, nh, dh, cond_dim, shape in ATTN_CASES:
        cls = SpatialAttention if kind == 'SpatialAttention' else TemporalAttention
        m = cls(n_head=nh, d_head=dh, embed=False, causal=cls is TemporalAttention,
                **({'key_dim': cond_dim} if cond_dim else {}))
        sd = MG.load_det(m)
        assert not any(k.endswith('freq') for k in sd), sorted(sd)
        x, cond = inputs(tag, shape, 1, cond_dim)
        x.requires_grad_(True)
        y = m(x, cond=cond)
        rec = check_case(m, sd, y, x, lambda s, xo: attn_oracle(s, kind, xo, nh, cond), tag)
        out[tag] = {'cls': kind, 'n_head': nh, 'd_head': dh, 'key_dim': cond_dim, 'shape': shape, **rec}


def gen_blocks(out):
    for tag, nh, dh, embed, transpose, cond_dim, shape in ST_CASES:
        kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
        m = SpaceTimeAttention(n_head=nh, d_head=dh, embed=embed, transpose=transpose, **kw)
        sd = MG.load_det(m)
        x, cond = inputs(tag, shape, 2 if transpose else 1, cond_dim)
        x.requires_grad_(True)
        y = m(x, cond=(None, cond)) if cond_dim else m(x)
        rec = check_case(m, sd, y, x, lambda s, xo: st_oracle(s, xo, nh, transpose, cond), tag)
        out[tag] = {'n_head': nh, 'd_head': dh, 'embed': embed, 'transpose': transpose, 'key_dim': cond_dim,
                    'shape': shape, **rec}


def gen_dynamics(out):
    dm = DynamicsModel(desc=fx.bp(DYN_DESC), **DYN)
    sd = MG.load_det(dm)
    assert not any(k.endswith('freq') for k in sd), sorted(sd)
    u = O.det_uniform('noembed.dyn.tokens', DYN_TOKENS_SHAPE) / (3 ** 0.5)            # in (-1, 1)
    tokens = ((u + 1) * 0.5 * DYN['tok_vocab']).long().clamp(0, DYN['tok_vocab'] - 1)
    ua = O.det_uniform('noembed.dyn.act', DYN_TOKENS_SHAPE[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * DYN['act_vocab']).long().clamp(0, DYN['act_vocab'] - 1)
    mask = O.det_uniform('noembed.dyn.mask', DYN_TOKENS_SHAPE) / (3 ** 0.5) < 0.5     # ~75 % masked
    logits, _ = dm(tokens, act)
    osd = identity_embed(sd)
    MG.close(O.dynamics_forward(osd, DYN_DESC, tokens, act), logits, 'Dynamics logits', rtol=2e-4, atol=2e-5)
    loss = dm.compute_loss(tokens, act, mask=mask)
    loss.backward()
    grads = MG.grads_of(dm)
    ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
    oloss = O.dynamics_loss(identity_embed(ref), DYN_DESC, tokens, act, mask)
    oloss.backward()
    MG.close(oloss, loss, 'Dynamics loss', rtol=2e-4)
    for k, g in grads.items():
        MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
    out['dynamics'] = {'desc': DYN_DESC, 'kw': DYN, 'tokens': tokens, 'act': act, 'mask': mask,
                       'keys': {k: tuple(v.shape) for k, v in sd.items()}, 'logits_shape': tuple(logits.shape),
                       'logits': sample('noembed.dyn.logits', logits, N_OUT), 'loss': loss.item(),
                       **grad_record('noembed.dyn.g', grads)}


def main():
    out = {}
    gen_attention(out)
    gen_blocks(out)
    gen_dynamics(out)
    path = os.path.join(MG.OUT, 'attn_noembed.pt')
    torch.save(out, path)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
