"""oracle/make_golden_ffn.py — tests/golden/st_block_ffn.pt by RUNNING THE REAL REFERENCE.   TEST INFRASTRUCTURE.

    OPEN_GENIE_REFERENCE=/path/to/open-genie python oracle/make_golden_ffn.py

SpaceTimeAttention(n_head=2, d_head=64) with the feed-forward options of the reference's ForwardBlock (hid_dim, d_out,
bias, kernel_size), run as oracle/make_golden.py runs its blocks: unmodified reference modules, closed-form weights and
inputs, CPU fp32, loss = mean(y^2). Every output and gradient is compared with oracle/ffn_oracle.py (a mismatch aborts);
the two variants the reference cannot run must raise there. Stored per case, to keep the file small: state_dict shapes,
every gradient's norm, and samples at oracle.genie_oracle.det_indices positions of y, dx and each gradient.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG                    # noqa: E402  (puts the reference and this repository on sys.path)
from make_golden import SpaceTimeAttention  # noqa: E402  (the reference's)

from oracle import ffn_oracle as FO         # noqa: E402
from oracle import genie_oracle as O        # noqa: E402

# (tag, constructor kwargs, key_dim or None, input shape)
CASES = (
    ('hid512', {'hid_dim': 512}, None, (2, 2, 4, 4, 128)),
    ('hid256_384_t1', {'hid_dim': (256, 384), 'transpose': True}, None, (2, 128, 2, 4, 4)),
    ('dout256_t1', {'d_out': 256, 'transpose': True}, None, (2, 128, 2, 4, 4)),
    ('dout256_hid512_t1', {'d_out': 256, 'hid_dim': 512, 'transpose': True}, None, (2, 128, 2, 4, 4)),
    ('bias', {'bias': True}, None, (2, 2, 4, 4, 128)),
    ('bias_cond', {'bias': True}, 4, (2, 2, 4, 4, 128)),
    ('bias_hid256_cond_t1', {'bias': True, 'hid_dim': 256, 'transpose': True}, 4, (2, 128, 2, 4, 4)),
    ('hid512_k1', {'hid_dim': 512, 'kernel_size': 1}, None, (2, 2, 4, 4, 128)),
)
N_OUT, N_GRAD = 256, 32          # sampled elements of y / dx, and of each gradient


def sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)].clone()


def inputs(tag, kw, cond_dim, shape):
    x = O.det_uniform(f'stffn.x.{tag}', shape)
    t = shape[2] if kw.get('transpose', False) else shape[1]
    cond = O.det_uniform(f'stffn.cond.{tag}', (shape[0], t, cond_dim)).sign() if cond_dim else None
    return x, cond


def main():
    out = {}
    for tag, kw, cond_dim, shape in CASES:
        kw = dict(kw, time_attn_kw={'key_dim': cond_dim}) if cond_dim else dict(kw)
        m = SpaceTimeAttention(n_head=2, d_head=64, **kw)
        sd = MG.load_det(m)
        transpose = kw.get('transpose', False)
        x, cond = inputs(tag, kw, cond_dim, shape)
        x.requires_grad_(True)
        y = m(x, cond=(None, cond)) if cond_dim else m(x)
        y.square().mean().backward()
        grads = MG.grads_of(m)
        ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
        xo = x.detach().clone().requires_grad_(True)
        yo = FO.spacetime_attention(ref, '', xo, 2, transpose, cond)
        yo.square().mean().backward()
        MG.close(yo, y, f'SpaceTimeAttention {tag}', rtol=2e-4, atol=2e-5)
        MG.close(xo.grad, x.grad, f'  dx {tag}', rtol=2e-4, atol=1e-6)
        for k, g in grads.items():
            MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
        names = sorted(grads)
        out[tag] = {'kw': kw, 'shape': shape, 'keys': {k: tuple(v.shape) for k, v in sd.items()},
                    'y_shape': tuple(y.shape), 'y': sample(f'stffn.y.{tag}', y, N_OUT),
                    'dx': sample(f'stffn.dx.{tag}', x.grad, N_OUT),
                    'grad_names': names, 'grad_norm': {k: grads[k].norm().item() for k in names},
                    'grad': torch.cat([sample(f'stffn.g.{tag}.{k}', grads[k], N_GRAD) for k in names])}
    for what, kw, shape in (('d_out=256, transpose=False', {'d_out': 256}, (1, 2, 4, 4, 128)),
                            ('d_inp=64', {'d_inp': 64}, (1, 2, 4, 4, 64))):
        try:
            SpaceTimeAttention(n_head=2, d_head=64, **kw)(torch.zeros(shape))
        except RuntimeError as e:
            print(f'  reference refuses SpaceTimeAttention({what}): ok  ({str(e).splitlines()[0][:60]})')
        else:
            raise AssertionError(f'the reference ran SpaceTimeAttention({what})')
    path = os.path.join(MG.OUT, 'st_block_ffn.pt')
    torch.save(out, path)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
