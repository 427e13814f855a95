"""Causal spatial and bidirectional temporal attention: `causal=` in SpatialAttention and TemporalAttention, through
og_flash_attn_causal_fwd / bwd (csrc/flash_attn.cu, kCausal) and og_temporal_attn_bidir_fwd / bwd
(csrc/temporal_attn_long.cu, kCausal off), and the modules built on them.

Kernel level: every output element against float64 (`drop_ref` / `drop_err` of test_gpu_attention_dropout, with the
causal mask on or off; at p = 0 the mask is all ones and they are attn_ref / attn_err), in guarded buffers. The
bidirectional kernels read inputs followed by NaN, so a key past T that entered any sum would show. Causality is
checked bit for bit. Model level: the modules against oracle.causal_attn_oracle and tests/golden/attn_causal.pt
(oracle/make_golden_causal_attn.py, from the unmodified reference). Which kernels run is pinned by name.
"""
import contextlib
import ctypes
import inspect

import pytest
import torch

from helpers import Guarded, det_weights, rel_l2
from oracle import causal_attn_oracle as CO
from oracle import genie_oracle as O
from oracle.noembed_oracle import identity_embed
from test_gpu_attention_dropout import _seed_tensor, drop_err, drop_ref, keep_mask
from test_gpu_attention_paths import (BF16, DEV, F32T, SLACK, U, _call, _kernels_run, _kvseq, _kvsum, _rand, _tseq,
                                      _tunseq, bf16_tol, check_all, gam)

GPU = pytest.mark.gpu
GOLDEN = 'attn_causal.pt'
SEED = 0x0DDC0FFEE1234567


# ------------------------------------------------------------------------------------------------------------------
# CPU: defaults, entry-point checks, the oracle against the golden
# ------------------------------------------------------------------------------------------------------------------
def test_causal_defaults_follow_the_reference():
    from open_genie_b200 import ops
    from open_genie_b200.module import get_module
    from open_genie_b200.module.attention import SpaceTimeAttention, SpatialAttention, TemporalAttention
    assert SpatialAttention(n_head=4, d_head=64).causal is False
    assert TemporalAttention(n_head=4, d_head=64).causal is False
    assert get_module('time_attn')(n_head=4, d_head=64).causal is False
    assert get_module('space_attn')(n_head=4, d_head=64, causal=True).causal is True
    st = SpaceTimeAttention(n_head=4, d_head=64)
    assert st.space_attn.causal is False and st.temp_attn.causal is True
    # the functional wrappers keep the calls made before the flag
    assert inspect.signature(ops.space_attention_res).parameters['causal'].default is False
    assert inspect.signature(ops.time_attention_res).parameters['causal'].default is True
    # the state_dict does not depend on the flag
    for cls in (SpatialAttention, TemporalAttention):
        assert cls(n_head=2, d_head=64, causal=True).state_dict().keys() == cls(n_head=2, d_head=64).state_dict().keys()


def _lib_and_ptr():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    return lib, ctypes.addressof(buf)


def test_causal_entry_points_validate_arguments():
    """p = 0 needs no seed; p > 0 needs one and p < 1; otherwise the counterparts' checks, codes and messages."""
    lib, ptr = _lib_and_ptr()
    calls = {
        'flash_fwd': lambda p, sd, S=64, C=256: lib.og_flash_attn_causal_fwd(ptr, ptr, ptr, ptr, None, None, ptr, 1, S,
                                                                            C, 4, 1.0, p, sd, None),
        'flash_bwd': lambda p, sd, S=64, C=256: lib.og_flash_attn_causal_bwd(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr,
                                                                            ptr, ptr, 1, S, C, 4, 1.0, p, sd, None),
        'bidir_fwd': lambda p, sd, S=40, C=256: lib.og_temporal_attn_bidir_fwd(
            ptr + 1, ptr, ptr, ptr, None, None, ptr, 1, S, 4, C, 4, 1.0, 0, p, sd, None),
        'bidir_bwd': lambda p, sd, S=40, C=256: lib.og_temporal_attn_bidir_bwd(
            ptr + 1, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, None, 1, S, 4, C, 4, 1.0, 0, p, sd, None),
    }
    for name, call in calls.items():
        assert call(0.1, None) == -1 and b'null seed' in lib.og_last_error(), name
        for p in (-0.1, 1.0, 1.5, float('nan')):
            assert call(p, ptr) == -1 and b'[0, 1)' in lib.og_last_error(), (name, p)
    for p, sd in ((0.0, None), (0.0, ptr), (0.1, ptr)):
        assert calls['flash_fwd'](p, sd, S=0) == -1 and b'flash_attn_fwd: empty problem' in lib.og_last_error()
        assert calls['flash_bwd'](p, sd, C=96) == -1 and b'flash_attn_bwd: needs d_head' in lib.og_last_error()
        assert calls['bidir_fwd'](p, sd) == -1 and b'temporal_attn_long_fwd: q, k' in lib.og_last_error()
        assert calls['bidir_bwd'](p, sd, C=96) == -2 and b'temporal_attn_long_bwd: d_head=24' in lib.og_last_error()
    assert lib.og_flash_attn_causal_fwd(None, ptr, ptr, ptr, None, None, ptr, 1, 64, 256, 4, 1.0, 0.0, None, None) == -1
    assert b'null pointer' in lib.og_last_error()
    assert lib.og_temporal_attn_bidir_bwd(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, None, None, None, 1, 40, 4, 256,
                                          4, 1.0, 0, 0.0, None, None) == -1
    assert b'missing dk/dv' in lib.og_last_error()


def _golden_module(c):
    from open_genie_b200.module.attention import SpatialAttention, TemporalAttention
    kw = {'key_dim': c['key_dim']} if c['key_dim'] else {}
    if c['cls'] == 'SpatialAttention':
        return SpatialAttention(n_head=c['n_head'], d_head=c['d_head'], embed=c['embed'], causal=True,
                                transpose=c['transpose'])
    return TemporalAttention(n_head=c['n_head'], d_head=c['d_head'], embed=c['embed'], transpose=c['transpose'], **kw)


def _golden_inputs(tag, c):
    shape = c['shape']
    x = O.det_uniform(f'causal.x.{tag}', shape)
    t = shape[2] if c['transpose'] else shape[1]
    cond = O.det_uniform(f'causal.cond.{tag}', (shape[0], t, c['key_dim'])).sign() if c['key_dim'] else None
    return x, cond


def _golden_oracle(sd, x, c, cond):
    sd = identity_embed(sd)
    if c['cls'] == 'SpatialAttention':
        return CO.spatial_attention(sd, '', x, c['n_head'], c['transpose'], causal=True)
    return CO.temporal_attention(sd, '', x, c['n_head'], c['transpose'], causal=False, cond=cond)


def _sample(key, t, n):
    return t.detach().float().cpu().flatten()[O.det_indices(key, t.numel(), n)]


def _golden_tags():
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', GOLDEN)
    return tuple(torch.load(path, weights_only=False))


TAGS = _golden_tags()


def test_golden_causal_covers_both_modules():
    assert {t.split('_')[0] for t in TAGS} == {'space', 'time'}
    assert {t.split('_')[1] for t in TAGS} == {'d16', 'd64', 'd128'}
    assert any(t.endswith('_c4') for t in TAGS) and any(t.endswith('_t1') for t in TAGS)
    assert any('_e0' in t for t in TAGS) and any('_e1' in t for t in TAGS)


@pytest.mark.parametrize('tag', TAGS)
def test_golden_causal_oracle(golden, tag):
    """The oracle reproduces the reference's outputs and gradients (CPU fp32)."""
    c = golden(GOLDEN)[tag]
    m = _golden_module(c)
    sd = det_weights(m)
    assert {k: tuple(v.shape) for k, v in sd.items()} == c['keys']
    x, cond = _golden_inputs(tag, c)
    ref = {k: v.clone().requires_grad_(k in c['grad_names']) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    y = _golden_oracle(ref, xo, c, cond)
    y.square().mean().backward()
    n = c['y'].numel()
    torch.testing.assert_close(_sample(f'causal.y.{tag}', y, n), c['y'], rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(_sample(f'causal.dx.{tag}', xo.grad, n), c['dx'], rtol=2e-4, atol=1e-6)
    for k in c['grad_names']:
        torch.testing.assert_close(_sample(f'causal.g.{tag}.{k}', ref[k].grad, 32), c['grad'][k], rtol=2e-4, atol=1e-6)
    if cond is not None:
        # With q = k = v (no key_dim) the scaled self-score |q|^2 scale dominates every row of these modules, so the
        # flag moves their outputs by 1e-4 .. 5e-2 only; causality itself is checked exactly at kernel level. With K / V
        # from the conditioning, the other flag's result is far from the reference's.
        flip = CO.temporal_attention(identity_embed(sd), '', x, c['n_head'], c['transpose'], causal=True, cond=cond)
        assert rel_l2(_sample(f'causal.y.{tag}', flip, n), c['y']) > 0.1


# ------------------------------------------------------------------------------------------------------------------
# float64 expectations
# ------------------------------------------------------------------------------------------------------------------
def _expect(qs, ks, vs, dos, scale, causal, keep, p):
    r = drop_ref(qs, ks, vs, scale, keep, p, causal=causal, do=dos)
    return r, drop_err(qs, ks, vs, r, scale, dos)


def flash_causal_expect(q, k, v, do, res, nh, scale, keep, p):
    """{output: (reference, tolerance)} of og_flash_attn_causal_fwd / bwd on bf16 [nseq, S, C] inputs."""
    nseq, S, C = q.shape
    sp = lambda t: t.double().view(nseq, S, nh, C // nh).transpose(1, 2)
    un = lambda t: t.transpose(1, 2).reshape(nseq, S, C)
    r, e = _expect(sp(q), sp(k), sp(v), sp(do), scale, True, keep, p)
    out = {name: (un(r[name]), bf16_tol(un(e[name]), un(r[name]))) for name in ('o', 'dq', 'dk', 'dv')}
    out['out'] = out.pop('o')
    out['lse'] = (r['lse'], SLACK * e['lse'])
    if res is not None:
        orr = un(r['o']) + res.double()
        out['out_res'] = (orr, SLACK * (un(e['o']) + U * orr.abs()))
    return out


def bidir_expect(q, k, v, do, res, nh, scale, bcast, keep, p, dk_init=None, dv_init=None):
    """The same for og_temporal_attn_bidir_fwd / bwd: q, do, res [B, T, P, C]; k, v the same or [B, T, C]."""
    B, T, P, C = q.shape
    f = lambda t: t.double()
    qs, dos = _tseq(f(q), nh), _tseq(f(do), nh)
    ks, vs = (_kvseq(f(k), nh), _kvseq(f(v), nh)) if bcast else (_tseq(f(k), nh), _tseq(f(v), nh))
    r, e = _expect(qs, ks, vs, dos, scale, False, keep, p)
    o, eo = _tunseq(r['o']), _tunseq(e['o'])
    out = {'out': (o, bf16_tol(eo, o))}
    orr = o + f(res)
    out['out_res'] = (orr, SLACK * (eo + U * orr.abs()))
    out['lse'] = (r['lse'].permute(0, 2, 1, 3), SLACK * e['lse'].permute(0, 2, 1, 3))
    out['dq'] = (_tunseq(r['dq']), bf16_tol(_tunseq(e['dq']), _tunseq(r['dq'])))
    if bcast:
        for name, init in (('dk', dk_init), ('dv', dv_init)):
            ref = f(init) + _kvsum(r[name])
            tol = _kvsum(e[name]) + gam(P + 2) * (f(init).abs() + _kvsum(r[name].abs()))
            out[name + '_bcast'] = (ref, SLACK * tol)
    else:
        for name in ('dk', 'dv'):
            out[name] = (_tunseq(r[name]), bf16_tol(_tunseq(e[name]), _tunseq(r[name])))
    return out


def test_bidir_expectation_rejects_a_causal_kernel():
    """The bidirectional bounds reject causal results, and the causal bounds reject non-causal ones."""
    B, T, P, nh, d = 1, 20, 2, 2, 64
    C, scale = nh * d, nh * d ** -0.5
    g = torch.Generator().manual_seed(3)
    q, k, v, do, res = ((torch.randn((B, T, P, C), generator=g) * 0.5).to(BF16) for _ in range(5))
    ones = torch.ones(B, P, nh, T, T, dtype=torch.bool)
    ex = bidir_expect(q, k, v, do, res, nh, scale, 0, ones, 0.0)
    check_all({n: (t[0].float() if n == 'lse' else t[0].to(BF16)) for n, t in ex.items()}, ex)
    r = drop_ref(_tseq(q.double(), nh), _tseq(k.double(), nh), _tseq(v.double(), nh), scale, ones, 0.0, causal=True)
    with pytest.raises(AssertionError):
        check_all({'out': _tunseq(r['o']).to(BF16)}, ex)
    qf, kf, vf, dof, rf = (t[0].permute(1, 0, 2).contiguous() for t in (q, k, v, do, res))   # pixels as flash sequences
    exf = flash_causal_expect(qf, kf, vf, dof, rf, nh, scale, torch.ones(P, nh, T, T, dtype=torch.bool), 0.0)
    with pytest.raises(AssertionError):
        check_all({'out': ex['out'][0][0].permute(1, 0, 2).to(BF16)}, exf)


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level: causal flash attention
# ------------------------------------------------------------------------------------------------------------------
def _seed_args(p, seed):
    if p == 0:
        return None, ()
    t = _seed_tensor(seed)
    return t, (t,)


def flash_causal_run(nseq, S, nh, d, seed, p=0.0, amp=0.5, aliased=False, residual=True):
    C, scale = d * nh, nh * d ** -0.5
    q = _rand((nseq, S, C), seed, amp)
    k, v = (q, q) if aliased else (_rand((nseq, S, C), seed + 1, amp), _rand((nseq, S, C), seed + 2))
    res, do = _rand((nseq, S, C), seed + 3), _rand((nseq, S, C), seed + 4)
    G = 64 * C
    names = ('out', 'out_res', 'dq', 'dk', 'dv') if residual else ('out', 'dq', 'dk', 'dv')
    outs = {n: Guarded(q.shape, BF16, G) for n in names}
    outs['lse'] = Guarded((nseq, nh, S), F32T, G)
    delta = Guarded((nseq, nh, S), F32T, G)
    st, _ = _seed_args(p, SEED + seed)
    sp = None if st is None else st.data_ptr()
    _call('og_flash_attn_causal_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(),
          res.data_ptr() if residual else None, outs['out_res'].ptr() if residual else None, outs['lse'].ptr(), nseq, S,
          C, nh, scale, p, sp)
    _call('og_flash_attn_causal_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), do.data_ptr(),
          outs['lse'].ptr(), delta.ptr(), outs['dq'].ptr(), outs['dk'].ptr(), outs['dv'].ptr(), nseq, S, C, nh, scale, p,
          sp)
    torch.cuda.synchronize()
    if p > 0:
        z = (torch.arange(nseq, device=DEV).view(nseq, 1) * nh + torch.arange(nh, device=DEV).view(1, nh))
        keep = keep_mask(SEED + seed, z, S, S, p)
    else:
        keep = torch.ones((nseq, nh, S, S), dtype=torch.bool, device=DEV)
    ex = flash_causal_expect(q, k, v, do, res if residual else None, nh, scale, keep, p)
    check_all({n: o.t for n, o in outs.items()}, ex)
    for n, o in list(outs.items()) + [('delta', delta)]:
        o.check_guard(n)


FLASH_S = [1, 2, 63, 64, 65, 200, 1024, 4096]


def _flash_geom(S, d):
    """(nseq, n_head): up to 16 heads on short sequences, fewer as S grows."""
    if S >= 4096:
        return 1, 1 if d == 128 else 2
    if S >= 1024:
        return 1, 4 if d == 16 else 2
    return 2, 16 if d == 16 else (8 if d == 64 else 3)


@GPU
@pytest.mark.parametrize('d', [16, 64, 128])
@pytest.mark.parametrize('S', FLASH_S)
def test_flash_causal_kernels(S, d):
    nseq, nh = _flash_geom(S, d)
    flash_causal_run(nseq, S, nh, d, seed=40000 + S + d)


@GPU
@pytest.mark.parametrize('d', [16, 64, 128])
@pytest.mark.parametrize('S', [65, 200])
def test_flash_causal_without_residual(S, d):
    flash_causal_run(3, S, 2, d, seed=41000 + S + d, residual=False)


@GPU
@pytest.mark.parametrize('d', [16, 64, 128])
def test_flash_causal_aliased_product_call(d):
    """q = k = v, as _SpaceAttnFn makes the call."""
    flash_causal_run(2, 130, 2, d, seed=42000 + d, aliased=True)


@GPU
@pytest.mark.parametrize('d', [16, 64, 128])
@pytest.mark.parametrize('S', [63, 200, 1024])
def test_flash_causal_dropout(S, d):
    """p = 0.1 after the causal mask, against the Philox mask restated in test_gpu_attention_dropout."""
    flash_causal_run(2 if S < 1024 else 1, S, 2, d, seed=43000 + S + d, p=0.1)


@GPU
@pytest.mark.parametrize('d', [16, 64, 128])
def test_flash_causality_is_exact(d):
    """Changing keys and values j > i0 leaves out, lse and dQ rows <= i0 bit-identical; changing queries and dO rows
    i < j0 leaves dK and dV rows >= j0 bit-identical."""
    nseq, S, nh = 2, 200, 2
    C, scale = d * nh, nh * d ** -0.5
    q, k, v, do = (_rand((nseq, S, C), 44000 + d + i) for i in range(4))

    def run(q, k, v, do):
        o, lse = torch.empty_like(q), torch.empty((nseq, nh, S), dtype=F32T, device=DEV)
        delta = torch.empty_like(lse)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
        _call('og_flash_attn_causal_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), None, None,
              lse.data_ptr(), nseq, S, C, nh, scale, 0.0, None)
        _call('og_flash_attn_causal_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
              lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), nseq, S, C, nh, scale,
              0.0, None)
        torch.cuda.synchronize()
        return o, lse, dq, dk, dv

    base = run(q, k, v, do)
    i0 = 100                       # inside the second tile, off its edge
    k2, v2 = k.clone(), v.clone()
    k2[:, i0 + 1:] = _rand(k2[:, i0 + 1:].shape, 44100, 3.0)
    v2[:, i0 + 1:] = _rand(v2[:, i0 + 1:].shape, 44101, 3.0)
    o, lse, dq, _, _ = run(q, k2, v2, do)
    assert torch.equal(o[:, :i0 + 1], base[0][:, :i0 + 1])
    assert torch.equal(lse[..., :i0 + 1], base[1][..., :i0 + 1])
    assert torch.equal(dq[:, :i0 + 1], base[2][:, :i0 + 1])
    assert not torch.equal(o[:, i0 + 1:], base[0][:, i0 + 1:])
    j0 = 90
    q2, do2 = q.clone(), do.clone()
    q2[:, :j0] = _rand(q2[:, :j0].shape, 44102, 3.0)
    do2[:, :j0] = _rand(do2[:, :j0].shape, 44103, 3.0)
    _, _, _, dk, dv = run(q2, k, v, do2)
    assert torch.equal(dk[:, j0:], base[3][:, j0:])
    assert torch.equal(dv[:, j0:], base[4][:, j0:])
    assert not torch.equal(dk[:, :j0], base[3][:, :j0])


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level: bidirectional tiled temporal attention
# ------------------------------------------------------------------------------------------------------------------
def _poisoned(x, extra):
    """x followed by `extra` NaN elements in one buffer: a read past the end of x turns an output into NaN."""
    buf = torch.full((x.numel() + extra,), float('nan'), dtype=x.dtype, device=x.device)
    buf[:x.numel()] = x.flatten()
    return buf[:x.numel()].view(x.shape)


def bidir_run(B, T, P, nh, d, bcast, seed, p=0.0, amp=1.0, aliased=False):
    """og_temporal_attn_bidir_fwd (with a residual) and og_temporal_attn_bidir_bwd on guarded outputs; the inputs are
    followed by 64 rows of NaN, the rows a last key tile would hold past T."""
    C, scale = nh * d, nh * d ** -0.5
    q = _poisoned(_rand((B, T, P, C), seed, amp), 64 * P * C)
    if aliased:
        k = v = q
    else:
        kvshape = (B, T, C) if bcast else (B, T, P, C)
        pitch = C if bcast else P * C
        k = _poisoned(_rand(kvshape, seed + 1, amp), 64 * pitch)
        v = _poisoned(_rand(kvshape, seed + 2), 64 * pitch)
    res = _rand((B, T, P, C), seed + 3)
    do = _poisoned(_rand((B, T, P, C), seed + 4), 64 * P * C)
    G = 64 * C
    outs = {n: Guarded(q.shape, BF16, G) for n in ('out', 'out_res', 'dq')}
    outs['lse'] = Guarded((B, nh, P, T), F32T, G)
    delta = Guarded((B, nh, P, T), F32T, G)
    st, _ = _seed_args(p, SEED + seed)
    sp = None if st is None else st.data_ptr()
    _call('og_temporal_attn_bidir_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), res.data_ptr(),
          outs['out_res'].ptr(), outs['lse'].ptr(), B, T, P, C, nh, scale, int(bcast), p, sp)
    dk_init = dv_init = None
    if bcast:
        dk_init, dv_init = _rand((B, T, C), seed + 5).float(), _rand((B, T, C), seed + 6).float()
        outs['dk_bcast'] = Guarded((B, T, C), F32T, G, dk_init)
        outs['dv_bcast'] = Guarded((B, T, C), F32T, G, dv_init)
        dks = (None, None, outs['dk_bcast'].ptr(), outs['dv_bcast'].ptr())
    else:
        outs['dk'], outs['dv'] = Guarded(q.shape, BF16, G), Guarded(q.shape, BF16, G)
        dks = (outs['dk'].ptr(), outs['dv'].ptr(), None, None)
    _call('og_temporal_attn_bidir_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), do.data_ptr(),
          outs['lse'].ptr(), delta.ptr(), outs['dq'].ptr(), *dks, B, T, P, C, nh, scale, int(bcast), p, sp)
    torch.cuda.synchronize()
    if p > 0:
        z = ((torch.arange(B, device=DEV).view(B, 1, 1) * P + torch.arange(P, device=DEV).view(1, P, 1)) * nh +
             torch.arange(nh, device=DEV).view(1, 1, nh))
        keep = keep_mask(SEED + seed, z, T, T, p)
    else:
        keep = torch.ones((B, P, nh, T, T), dtype=torch.bool, device=DEV)
    ex = bidir_expect(q, k, v, do, res, nh, scale, bcast, keep, p, dk_init, dv_init)
    check_all({n: o.t for n, o in outs.items()}, ex)
    for n, o in list(outs.items()) + [('delta', delta)]:
        o.check_guard(n)


BIDIR_T = [1, 2, 15, 16, 17, 32, 33, 64, 65, 200, 1024]


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('d', [16, 64, 128])
@pytest.mark.parametrize('T', BIDIR_T)
def test_bidir_kernels(T, d, bcast):
    """One sequence per batch (B = 1), so the NaN rows follow the clip's last frame directly."""
    P, nh = (3, 2) if T >= 1024 else (5, 2)
    bidir_run(1, T, P, nh, d, bcast, seed=50000 + 10 * T + d + bcast)


@GPU
@pytest.mark.parametrize('d', [16, 64, 128])
def test_bidir_two_clips_and_aliased_call(d):
    """B = 2 (the rows past the first clip's T are the second clip's) and q = k = v as _TimeAttnFn calls it."""
    bidir_run(2, 70, 4, 2, d, 0, seed=51000 + d, aliased=True)
    bidir_run(2, 40, 4, 2, d, 1, seed=51500 + d)


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('d', [16, 64, 128])
@pytest.mark.parametrize('T', [16, 65])
def test_bidir_dropout(T, d, bcast):
    bidir_run(1, T, 4, 2, d, bcast, seed=52000 + T + d + bcast, p=0.1)


@GPU
def test_bidir_bcast_gradient_many_pixel_chunks():
    """kv_bcast = 1 at P = 2048: the dK / dV kernel's chunked path with its atomic flush, over all query tiles."""
    bidir_run(1, 70, 2048, 2, 64, 1, seed=53000)


# ------------------------------------------------------------------------------------------------------------------
# GPU, modules: kernel names, the golden, the oracle, a graph replay
# ------------------------------------------------------------------------------------------------------------------
def _module_step(m, shape, seed, cond_dim=None):
    def run():
        x = O.det_uniform(f'causal.names.{seed}', shape).to(DEV).requires_grad_(True)
        cond = None
        if cond_dim:
            cond = O.det_uniform(f'causal.names.c.{seed}', (shape[0], shape[1], cond_dim)).to(DEV)
        y = m(x, cond=cond) if cond_dim else m(x)
        y.float().square().mean().backward()
    return run


def _has(names, kernel):
    return any(kernel in n for n in names)


@GPU
def test_kernel_names_of_the_new_configurations():
    from open_genie_b200.module.attention import SpatialAttention, TemporalAttention
    m = SpatialAttention(n_head=2, d_head=64, causal=True).to(DEV)
    names = _kernels_run(_module_step(m, (1, 2, 9, 9, 128), 1))
    assert _has(names, 'og_flash_attn_causal_fwd_kernel') and _has(names, 'og_flash_attn_causal_bwd_kernel')
    assert not _has(names, 'og_flash_attn_fwd_kernel') and not _has(names, 'og_flash_attn_bwd_kernel')
    for T, cond_dim in ((16, None), (16, 4), (40, None)):       # T <= 32 at d = 64 too: never the per-pixel kernels
        m = TemporalAttention(n_head=2, d_head=64, **({'key_dim': cond_dim} if cond_dim else {})).to(DEV)
        names = _kernels_run(_module_step(m, (1, T, 3, 3, 128), 2 + T, cond_dim))
        for k in ('og_temporal_attn_bidir_fwd_kernel', 'og_temporal_attn_bidir_bwd_dq_kernel',
                  'og_temporal_attn_bidir_bwd_dkdv_kernel'):
            assert _has(names, k), (T, k)
        assert not _has(names, 'og_temporal_attn_fwd') and not _has(names, 'og_temporal_attn_long_fwd_kernel')


@GPU
def test_spacetime_and_causal_temporal_keep_their_kernels():
    from open_genie_b200.module.attention import SpaceTimeAttention, TemporalAttention
    m = SpaceTimeAttention(n_head=2, d_head=64).to(DEV)
    names = _kernels_run(_module_step(m, (1, 16, 3, 3, 128), 3))
    assert _has(names, 'og_flash_attn_fwd_kernel') and _has(names, 'og_temporal_attn_fwd_mma_kernel')
    assert not any(_has(names, k) for k in ('causal_fwd_kernel', 'causal_bwd_kernel', 'bidir'))
    m = TemporalAttention(n_head=2, d_head=64, causal=True).to(DEV)
    names = _kernels_run(_module_step(m, (1, 40, 3, 3, 128), 4))
    assert _has(names, 'og_temporal_attn_long_fwd_kernel') and not _has(names, 'bidir')


@GPU
@pytest.mark.parametrize('tag', TAGS)
def test_golden_causal_on_gpu(golden, tag):
    """The modules against the reference's own outputs and gradients, with the tolerances of the stand-alone modules of
    test_gpu_attention_noembed (their output is bf16(x + attention(x)) - x)."""
    c = golden(GOLDEN)[tag]
    m = _golden_module(c)
    det_weights(m)
    m.to(DEV)
    x, cond = _golden_inputs(tag, c)
    xg = x.to(DEV).requires_grad_(True)
    y = m(xg, cond=cond.to(DEV)) if cond is not None else m(xg)
    y.float().square().mean().backward()
    n = c['y'].numel()
    assert rel_l2(_sample(f'causal.y.{tag}', y, n), c['y']) < 6e-2
    assert rel_l2(_sample(f'causal.dx.{tag}', xg.grad, n), c['dx']) < 6e-2
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k in c['grad_names']:
        got = _sample(f'causal.g.{tag}.{k}', grads[k], 32)
        assert rel_l2(got, c['grad'][k]) < 0.1, (k, rel_l2(got, c['grad'][k]))
        assert abs(grads[k].float().norm().item() - c['grad_norm'][k]) <= 0.05 * c['grad_norm'][k] + 1e-6, k


@GPU
@pytest.mark.parametrize('p', [0.0, 0.1])
@pytest.mark.parametrize('nh,dh', [(4, 16), (2, 64), (1, 128)])
def test_modules_against_oracle(nh, dh, p):
    """Longer sequences than the golden's (S = 200, T = 40 and 70) against the oracle; with dropout the oracle takes
    the masks of the seeds the modules drew."""
    from open_genie_b200.module.attention import SpatialAttention, TemporalAttention
    from test_gpu_attention_dropout import _values, oracle_with_seeds, recorded_seeds
    C = nh * dh
    for kind, shape in (('space', (1, 2, 10, 20, C)), ('time', (1, 40, 3, 3, C)), ('time', (1, 70, 2, 2, C))):
        m = (SpatialAttention(n_head=nh, d_head=dh, causal=True, dropout=p) if kind == 'space'
             else TemporalAttention(n_head=nh, d_head=dh, dropout=p))
        sd = det_weights(m)
        m.to(DEV)
        tag = f'causal.mod.{kind}.{nh}.{shape[1]}'
        x = O.det_uniform(tag + '.x', shape)
        gy = O.det_uniform(tag + '.gy', shape, 1e-3)
        xg = x.to(DEV).requires_grad_(True)
        with recorded_seeds() as seeds:
            y = m(xg)
        (y.float() * gy.to(DEV)).sum().backward()
        ref = {k: v.clone().requires_grad_(k.startswith('norm.')) for k, v in sd.items()}
        xr = x.clone().requires_grad_(True)
        assert len(seeds) == (1 if p > 0 else 0)
        with oracle_with_seeds(_values(seeds), p) if p > 0 else contextlib.nullcontext([]) as left:
            if kind == 'space':
                yr = CO.spatial_attention(ref, '', xr, nh, False, causal=True)
            else:
                yr = CO.temporal_attention(ref, '', xr, nh, False, causal=False)
        assert not left
        (yr * gy).sum().backward()
        assert rel_l2(y.float().cpu(), yr.detach()) < 6e-2, (kind, shape)
        assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2, (kind, shape)
        for k in ('norm.weight', 'norm.bias'):
            got = dict(m.named_parameters())[k].grad.float().cpu()
            assert rel_l2(got, ref[k].grad) < 8e-2, (kind, shape, k)


class _CausalStep(torch.nn.Module):
    """A causal SpatialAttention and a bidirectional TemporalAttention as a GraphedTrainStep model."""

    def __init__(self):
        super().__init__()
        from open_genie_b200.module.attention import SpatialAttention, TemporalAttention
        self.space = SpatialAttention(n_head=2, d_head=64, causal=True)
        self.time = TemporalAttention(n_head=2, d_head=64)
        self.w = O.det_uniform('causal.graph.w', (2, 16, 4, 4, 128)).to(DEV)

    def training_step(self, batch, batch_idx):
        x = self.space(batch, _residual=True)
        return (self.time(x, _residual=True).float() * self.w).mean()


@GPU
def test_graphed_train_step_with_causal_modules_matches_eager():
    from open_genie_b200.graph import GraphedTrainStep
    from open_genie_b200.optim import FusedAdamW
    model = _CausalStep()
    det_weights(model.space)
    det_weights(model.time)
    model.to(DEV)
    opt = FusedAdamW(model.parameters(), lr=0.0, weight_decay=0.0)
    x = O.det_uniform('causal.graph.x', (2, 16, 4, 4, 128)).to(DEV)
    step = GraphedTrainStep(model, opt, x)
    grads = lambda: {k: p.grad.float().cpu().clone() for k, p in model.named_parameters() if p.grad is not None}
    results = []
    for _ in range(2):
        loss = step(x)
        torch.cuda.synchronize()
        results.append((loss.item(), grads()))
    model.zero_grad(set_to_none=True)
    eager = model.training_step(x, 0)
    eager.backward()
    g_e = grads()
    del step
    torch.cuda.synchronize()
    assert len(g_e) == 4
    for l, g in results:
        assert abs(eager.item() - l) <= 1e-3 * abs(l) + 1e-7, (eager.item(), l)
        assert sorted(g) == sorted(g_e)
        for k in g:
            assert rel_l2(g[k], g_e[k]) < 1e-3, (k, rel_l2(g[k], g_e[k]))
