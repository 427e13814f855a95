"""oracle/make_golden_causal_attn.py — tests/golden/attn_causal.pt by RUNNING THE REAL REFERENCE.   TEST INFRASTRUCTURE.

    OPEN_GENIE_REFERENCE=/path/to/open-genie python oracle/make_golden_causal_attn.py

The two stand-alone attention configurations whose `causal` differs from SpaceTimeAttention's: SpatialAttention(
causal=True) (SDPA is_causal=True over the h*w tokens in raster order) and a bare TemporalAttention (the reference's
default causal=False: bidirectional over t), run as oracle/make_golden.py runs its models: unmodified reference modules,
closed-form weights and inputs, CPU fp32. Every result is compared with oracle.causal_attn_oracle (genie_oracle's
attention_core with the flag; oracle.noembed_oracle.identity_embed for embed=False); a mismatch aborts. Cases: both
modules at d_head 16 (4 heads), 64 (2 heads) and 128 (1 head), with embed True and False, the temporal one with and
without a key_dim = 4 conditioning, and one transposed input of each. The modules' outputs (no skip); loss = mean(y^2).
Stored per case: the configuration, every gradient's norm, and samples at oracle.genie_oracle.det_indices positions of
the output, dx and each gradient.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG                    # noqa: E402  (puts the reference and this repository on sys.path)
import torch                                # noqa: E402
from genie.module.attention import SpatialAttention, TemporalAttention  # noqa: E402  (the reference's)

from oracle import causal_attn_oracle as CO  # noqa: E402
from oracle import genie_oracle as O        # noqa: E402
from oracle.noembed_oracle import identity_embed  # noqa: E402

WIDTHS = ((4, 16), (2, 64), (1, 128))       # (n_head, d_head)


def cases():
    """(tag, class name, n_head, d_head, embed, key_dim or None, transpose, input shape)"""
    out = []
    for nh, dh in WIDTHS:
        C = nh * dh
        for embed in (True, False):
            e = 'e1' if embed else 'e0'
            out.append((f'space_d{dh}_{e}', 'SpatialAttention', nh, dh, embed, None, False, (2, 2, 9, 9, C)))
            for kd in (None, 4):
                c = f'_c{kd}' if kd else ''
                out.append((f'time_d{dh}_{e}{c}', 'TemporalAttention', nh, dh, embed, kd, False, (2, 12, 3, 3, C)))
    out.append(('space_d64_e1_t1', 'SpatialAttention', 2, 64, True, None, True, (2, 128, 2, 9, 9)))
    out.append(('time_d64_e1_t1', 'TemporalAttention', 2, 64, True, None, True, (2, 128, 40, 2, 2)))
    return tuple(out)


CASES = cases()
N_OUT, N_GRAD = 256, 32          # sampled elements of an output, and of each gradient


def sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)].clone()


def oracle(kind, sd, x, nh, transpose, cond):
    sd = identity_embed(sd)
    if kind == 'SpatialAttention':
        return CO.spatial_attention(sd, '', x, nh, transpose, causal=True)
    return CO.temporal_attention(sd, '', x, nh, transpose, causal=False, cond=cond)


def gen(out):
    for tag, kind, nh, dh, embed, kd, transpose, shape in CASES:
        if kind == 'SpatialAttention':
            m = SpatialAttention(n_head=nh, d_head=dh, embed=embed, causal=True, transpose=transpose)
        else:
            m = TemporalAttention(n_head=nh, d_head=dh, embed=embed, transpose=transpose,
                                  **({'key_dim': kd} if kd else {}))
            assert m.causal is False
        sd = MG.load_det(m)
        x = O.det_uniform(f'causal.x.{tag}', shape)
        t_axis = 2 if transpose else 1
        cond = O.det_uniform(f'causal.cond.{tag}', (shape[0], shape[t_axis], kd)).sign() if kd else None
        x.requires_grad_(True)
        y = m(x, cond=cond) if kd else m(x)
        y.square().mean().backward()
        grads = MG.grads_of(m)
        ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
        xo = x.detach().clone().requires_grad_(True)
        yo = oracle(kind, ref, xo, nh, transpose, cond)
        yo.square().mean().backward()
        MG.close(yo, y, tag, rtol=2e-4, atol=2e-5)
        MG.close(xo.grad, x.grad, f'  dx {tag}', rtol=2e-4, atol=1e-6)
        for k, g in grads.items():
            MG.close(ref[k].grad, g, f'  d {k}', rtol=2e-4, atol=1e-6)
        names = sorted(grads)
        out[tag] = {'cls': kind, 'n_head': nh, 'd_head': dh, 'embed': embed, 'key_dim': kd, 'transpose': transpose,
                    'shape': shape, 'keys': {k: tuple(v.shape) for k, v in sd.items()},
                    'y': sample(f'causal.y.{tag}', y, N_OUT), 'dx': sample(f'causal.dx.{tag}', x.grad, N_OUT),
                    'grad_names': names, 'grad_norm': {k: grads[k].norm().item() for k in names},
                    'grad': {k: sample(f'causal.g.{tag}.{k}', grads[k], N_GRAD) for k in names}}


def main():
    out = {}
    gen(out)
    path = os.path.join(MG.OUT, 'attn_causal.pt')
    torch.save(out, path)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
