"""Attention without a rotary embedding (embed=False): the LayerNorm-only row passes og_ln_rows_fwd / bwd
(csrc/attention_rows.cu), the autograd functions that call them with freq=None (ops._SpaceAttnFn, ops._TimeAttnFn) and
the modules built on them.

Kernel level: every output element against a float64 LayerNorm with the per-element bounds of
test_gpu_attention_paths (`rope_ln_ref` / `rope_ln_bwd_expect` at zero frequencies, where the rotation is the identity),
in guarded buffers, at C = 16 .. 1024 with aligned (vectorised kernels) and misaligned (one warp per row) pointers.
CPU tests show these bounds reject a rotation left in, a missing gradient term and dgamma overwritten instead of
accumulated. Model level: the modules against the CPU oracle (oracle.noembed_oracle.identity_embed: genie_oracle at
zero frequencies) with the tolerances of the d_head = 16 / 128 model tests, and tests/golden/attn_noembed.pt
(oracle/make_golden_noembed.py, from the unmodified reference) pins the oracle, the state_dict keys and the modules.
"""
import ctypes

import pytest
import torch

from helpers import det_weights, rel_l2
from oracle import ffn_oracle
from oracle import fixtures as fx
from oracle import genie_oracle as O
from oracle.noembed_oracle import identity_embed
from test_gpu_attention_paths import (BF16, DEV, F32T, F_LN, Guarded, _bf, _call, _cpu_rand, _kernels_run, _rand,
                                      _rejects, _rot_t, _ln_bwd, bf16_tol, check_all, rope_ln_bwd_expect,
                                      rope_ln_ref)

GPU = pytest.mark.gpu
GOLDEN = 'attn_noembed.pt'
ATTN_CASES = ('spatial', 'temporal', 'temporal_c4')
ST_CASES = ('d16_e00', 'd16_e01', 'd16_e10', 'd16_e00_c4', 'd16_e00_t1', 'd64_e00', 'd64_e01', 'd64_e10', 'mixed_e01')
EMBEDS = (True, False, (False, True), (True, False))


# ------------------------------------------------------------------------------------------------------------------
# float64 reference: LayerNorm(x) is LayerNorm(RoPE(x)) at zero frequencies (cos 0 = 1, sin 0 = 0 exactly)
# ------------------------------------------------------------------------------------------------------------------
def ln_ref(x, gamma, beta):
    rows, C = x.shape
    return rope_ln_ref(x, torch.zeros(rows, dtype=torch.long, device=x.device), torch.zeros(C // 2), gamma, beta)


def ln_fwd_expect(st, gamma, beta):
    """{'y': (reference, tolerance)} of og_ln_rows_fwd: fp32 statistics (F_LN) and the final bf16 rounding."""
    y = st['y']
    tol = bf16_tol(F_LN * (gamma.double().abs().to(y.device) * (st['xh'].abs() + 1) +
                           beta.double().abs().to(y.device)), y)
    return {'y': (y, tol)}


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument checks, construction, state_dict keys, the oracle against the golden, the bounds reject mistakes
# ------------------------------------------------------------------------------------------------------------------
def _lib_and_ptr():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    return lib, ctypes.addressof(buf)


def test_ln_rows_argument_checks():
    """Every bad argument returns -1 with a message, before anything is launched (no device needed)."""
    lib, p = _lib_and_ptr()
    fwd = lambda x=p, g=p, b=p, y=p, rows=4, C=64: lib.og_ln_rows_fwd(x, g, b, 1e-5, y, rows, C, None)
    bwd = lambda x=p, g=p, g0=p, g1=None, g2=None, add=None, dx=p, dg=p, db=p, rows=4, C=64: lib.og_ln_rows_bwd(
        x, g, 1e-5, g0, g1, g2, add, dx, dg, db, rows, C, None)
    cases = [
        (fwd, dict(x=None), b'ln_rows_fwd: bad arguments'), (fwd, dict(g=None), b'bad arguments'),
        (fwd, dict(b=None), b'bad arguments'), (fwd, dict(y=None), b'bad arguments'),
        (fwd, dict(rows=0), b'bad arguments'), (fwd, dict(rows=-3), b'bad arguments'),
        (fwd, dict(C=63), b'C=63 must be even'), (fwd, dict(C=0), b'C=0 must be even'),
        (fwd, dict(C=-2), b'C=-2'), (fwd, dict(C=1026), b'C=1026'),
        (fwd, dict(x=p + 2), b'4-byte aligned'), (fwd, dict(y=p + 2), b'4-byte aligned'),
        (bwd, dict(x=None), b'ln_rows_bwd: bad arguments'), (bwd, dict(g=None), b'bad arguments'),
        (bwd, dict(g0=None), b'bad arguments'), (bwd, dict(dx=None), b'bad arguments'),
        (bwd, dict(dg=None), b'bad arguments'), (bwd, dict(db=None), b'bad arguments'),
        (bwd, dict(rows=0), b'bad arguments'), (bwd, dict(C=5), b'C=5 must be even'),
        (bwd, dict(C=2048), b'C=2048'), (bwd, dict(g1=p + 2), b'4-byte aligned'),
        (bwd, dict(g2=p + 6), b'4-byte aligned'), (bwd, dict(add=p + 2), b'4-byte aligned'),
        (bwd, dict(dx=p + 2), b'4-byte aligned'), (bwd, dict(dg=p + 2), b'dgamma and dbeta'),
    ]
    for fn, kw, msg in cases:
        assert fn(**kw) == -1, kw
        assert msg in lib.og_last_error(), (kw, lib.og_last_error())
    # the RoPE passes keep refusing a missing frequency table
    assert lib.og_rope_ln_fwd(p, None, p, p, 1e-5, p, 4, 64, 1, 4, None, None) == -1
    assert b'rope_ln_fwd: bad arguments' in lib.og_last_error()
    assert lib.og_rope_ln_bwd(p, None, p, 1e-5, p, None, None, None, p, p, p, 4, 64, 1, 4, None, None) == -1
    assert b'rope_ln_bwd: bad arguments' in lib.og_last_error()


@pytest.mark.parametrize('embed', EMBEDS, ids=str)
def test_every_embed_combination_builds(embed):
    import torch.nn as nn
    from open_genie_b200.module.attention import RotaryEmbedding, SpaceTimeAttention
    m = SpaceTimeAttention(n_head=4, d_head=16, embed=embed)
    es, et = (embed, embed) if isinstance(embed, bool) else embed
    for attn, e in ((m.space_attn, es), (m.temp_attn, et)):
        assert isinstance(attn.embed, RotaryEmbedding if e else nn.Identity)
        assert (attn._freq is None) == (not e)
    keys = set(m.state_dict())
    assert ('space_attn.embed.freq' in keys) == es and ('temp_attn.embed.freq' in keys) == et


def test_embed_true_is_unchanged():
    """The default keeps its rotary embedding: the frequencies the reference builds, as a state_dict entry, handed to
    the attention functions."""
    from open_genie_b200.module.attention import RotaryEmbedding, SpatialAttention, TemporalAttention
    for cls, kind in ((SpatialAttention, '2d'), (TemporalAttention, '1d')):
        for m in (cls(n_head=4, d_head=16), cls(n_head=4, d_head=16, embed=True)):
            assert isinstance(m.embed, RotaryEmbedding) and m._freq is m.embed.freq
            assert torch.equal(m.embed.freq, O.rope_freq(64, kind))
            assert sorted(m.state_dict()) == ['embed.freq', 'norm.bias', 'norm.weight']
        assert sorted(cls(n_head=4, d_head=16, embed=False).state_dict()) == ['norm.bias', 'norm.weight']


def test_blueprints_pass_embed():
    import open_genie_b200 as og
    from open_genie_b200.module.attention import Attention
    desc = (('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 16, 'embed': (False, True), 'transpose': False}),)
    dm = og.DynamicsModel(desc, tok_vocab=16, act_vocab=4, embed_dim=64)
    attns = [(n, m) for n, m in dm.named_modules() if isinstance(m, Attention)]
    assert len(attns) == 4
    for n, m in attns:
        assert (m._freq is None) == n.endswith('space_attn'), n


def test_identity_embed_completes_only_missing_frequencies():
    from open_genie_b200.module.attention import SpaceTimeAttention
    sd = det_weights(SpaceTimeAttention(n_head=4, d_head=16, embed=(False, True)))
    full = identity_embed(sd)
    assert torch.equal(full['space_attn.embed.freq'], torch.zeros(32))
    assert full['temp_attn.embed.freq'] is sd['temp_attn.embed.freq']
    x = _cpu_rand((3, 10, 64), 1).float()
    assert torch.equal(O.rope(x, full['space_attn.embed.freq']), x)


def _golden_module(c):
    from open_genie_b200.module.attention import SpaceTimeAttention, SpatialAttention, TemporalAttention
    if 'cls' in c:
        cls = SpatialAttention if c['cls'] == 'SpatialAttention' else TemporalAttention
        return cls(n_head=c['n_head'], d_head=c['d_head'], embed=False, causal=cls is TemporalAttention,
                   **({'key_dim': c['key_dim']} if c['key_dim'] else {}))
    kw = {'time_attn_kw': {'key_dim': c['key_dim']}} if c['key_dim'] else {}
    return SpaceTimeAttention(n_head=c['n_head'], d_head=c['d_head'], embed=c['embed'], transpose=c['transpose'], **kw)


def _golden_inputs(tag, c):
    shape = c['shape']
    x = O.det_uniform(f'noembed.x.{tag}', shape)
    t = shape[2] if c.get('transpose') else shape[1]
    cond = O.det_uniform(f'noembed.cond.{tag}', (shape[0], t, c['key_dim'])).sign() if c['key_dim'] else None
    return x, cond


def _golden_oracle(sd, x, c, cond):
    """genie_oracle on the completed state_dict; the mixed block composed from its parts."""
    import torch.nn.functional as F
    sd = identity_embed(sd)
    nh = c['n_head']
    if 'cls' in c:
        if c['cls'] == 'SpatialAttention':
            return O.spatial_attention(sd, '', x, nh, False)
        return O.temporal_attention(sd, '', x, nh, False, cond)
    if isinstance(nh, int):
        return O.spacetime_attention(sd, '', x, nh, c['transpose'], cond)
    x = O.spatial_attention(sd, 'space_attn.', x, nh[0], False) + x
    x = O.temporal_attention(sd, 'temp_attn.', x, nh[1], False, cond) + x
    y = F.group_norm(x.movedim(-1, 1), nh[1], sd['ffn.1.net.0.weight'], sd['ffn.1.net.0.bias'], 1e-5)
    return F.conv3d(y, sd['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x


def _sample(key, t, n):
    return t.detach().float().cpu().flatten()[O.det_indices(key, t.numel(), n)]


def _golden_grads(prefix, c, grads):
    return [(k, _sample(f'{prefix}.{k}', grads[k], 32), c['grad'][k], c['grad_norm'][k]) for k in c['grad_names']]


def _ref_sd(sd):
    return {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith(('freq', 'bit_mask')))
            for k, v in sd.items()}


def test_golden_noembed_holds_every_case(golden):
    g = golden(GOLDEN)
    assert tuple(g) == ATTN_CASES + ST_CASES + ('dynamics',)
    assert {g[t]['embed'] for t in ST_CASES} == {False, (False, True), (True, False)}
    assert g['dynamics']['desc'] == DYN_DESC and g['dynamics']['kw'] == DYN


@pytest.mark.parametrize('tag', ATTN_CASES + ST_CASES)
def test_golden_noembed_keys_and_oracle(golden, tag):
    """The module's state_dict keys are the reference's, and the CPU oracle reproduces the reference's outputs and
    gradients."""
    c = golden(GOLDEN)[tag]
    m = _golden_module(c)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == c['keys']
    sd = det_weights(m)
    ref = _ref_sd(sd)
    x, cond = _golden_inputs(tag, c)
    x.requires_grad_(True)
    y = _golden_oracle(ref, x, c, cond)
    y.square().mean().backward()
    n = c['y'].numel()
    torch.testing.assert_close(_sample(f'noembed.y.{tag}', y, n), c['y'], rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(_sample(f'noembed.dx.{tag}', x.grad, n), c['dx'], rtol=2e-4, atol=1e-6)
    grads = {k: v.grad for k, v in ref.items() if v.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads(f'noembed.g.{tag}', c, grads):
        torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-6)
        assert abs(grads[k].norm().item() - norm) <= 1e-4 * norm + 1e-7, k


DYN_DESC = (('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 16, 'transpose': False, 'embed': False}),)
DYN = dict(tok_vocab=16, act_vocab=4, embed_dim=64)


def test_golden_noembed_oracle_dynamics(golden):
    import open_genie_b200 as og
    c = golden(GOLDEN)['dynamics']
    dm = og.DynamicsModel(DYN_DESC, **DYN)
    assert {k: tuple(v.shape) for k, v in dm.state_dict().items()} == c['keys']
    ref = _ref_sd(det_weights(dm))
    logits = O.dynamics_forward(identity_embed(ref), DYN_DESC, c['tokens'], c['act'])
    assert tuple(logits.shape) == c['logits_shape']
    torch.testing.assert_close(_sample('noembed.dyn.logits', logits, c['logits'].numel()), c['logits'], rtol=2e-4,
                               atol=2e-5)
    loss = O.dynamics_loss(identity_embed(ref), DYN_DESC, c['tokens'], c['act'], c['mask'])
    loss.backward()
    assert abs(loss.item() - c['loss']) <= 2e-4 * abs(c['loss'])
    grads = {k: v.grad for k, v in ref.items() if v.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads('noembed.dyn.g', c, grads):
        torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-6)
        assert abs(grads[k].norm().item() - norm) <= 1e-4 * norm + 1e-7, k


def test_tolerances_reject_plausible_ln_rows_bugs():
    """An exactly right result (the float64 reference rounded once) passes; each mistake is rejected: a rotation left
    in (the '1d' and '2d' RoPE at the rows' positions), one of the gradient terms g1, g2 or `add` dropped, and dgamma /
    dbeta overwritten instead of accumulated."""
    rows, C = 40, 128
    x = _cpu_rand((rows, C), 400).double()
    gamma = 1 + 0.2 * torch.randn(C, generator=torch.Generator().manual_seed(2))
    beta = 0.2 * torch.randn(C, generator=torch.Generator().manual_seed(3))
    st = ln_ref(x, gamma, beta)
    ef = ln_fwd_expect(st, gamma, beta)
    check_all({'y': _bf(ef['y'][0])}, ef)
    g0, g1, g2, add = (_cpu_rand((rows, C), 401 + i).double() for i in range(4))
    dg0, db0 = _cpu_rand((C,), 405).double(), _cpu_rand((C,), 406).double()
    g = g0 + g1 + g2
    eb = rope_ln_bwd_expect(st, g, gamma, add, dg_init=dg0, db_init=db0)
    exact = {'dx': _bf(eb['dx'][0]), 'dgamma': eb['dgamma'][0].float(), 'dbeta': eb['dbeta'][0].float()}
    check_all(exact, eb)
    pos = torch.arange(rows) % 5
    for kind in ('1d', '2d'):
        rot = rope_ln_ref(x, pos, O.rope_freq(C, kind), gamma, beta)
        _rejects({'y': _bf(rot['y'])}, ef)
        _rejects({'dx': _bf(_rot_t(_ln_bwd(rot, g, gamma), rot) + add)}, eb)
    for partial in (g0 + g1, g0 + g2, g1 + g2):
        wrong = rope_ln_bwd_expect(st, partial, gamma, add, dg_init=dg0, db_init=db0)
        _rejects({'dx': _bf(wrong['dx'][0])}, eb)
        _rejects({'dgamma': wrong['dgamma'][0].float()}, eb)
    _rejects({'dx': _bf(eb['dx'][0] - add)}, eb)
    _rejects({'dgamma': (eb['dgamma'][0] - dg0).float()}, eb)
    _rejects({'dbeta': (eb['dbeta'][0] - db0).float()}, eb)


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level
# ------------------------------------------------------------------------------------------------------------------
def _params(C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return 1 + 0.2 * torch.randn(C, generator=g, device=DEV), 0.2 * torch.randn(C, generator=g, device=DEV)


def _place(t, offset):
    """A copy of t placed `offset` bf16 elements into its buffer: offset 2 (4 bytes) keeps the bf16x2 accesses of the
    one-warp-per-row kernels aligned and breaks the 16-byte alignment of the vectorised ones."""
    b = torch.empty(t.numel() + offset, dtype=BF16, device=DEV)
    b[offset:].copy_(t.flatten())
    return b[offset:].view(t.shape)


def ln_rows_run(rows, C, terms, offset, seed):
    """og_ln_rows_fwd and og_ln_rows_bwd on guarded outputs; `terms` names the gradient inputs given (g0 always)."""
    x, g0, g1, g2, add = (_rand((rows, C), seed + i) for i in range(5))
    gamma, beta = _params(C, seed + 5)
    dg0, db0 = _rand((C,), seed + 6).float(), _rand((C,), seed + 7).float()
    use = {'g1': g1 if 'g1' in terms else None, 'g2': g2 if 'g2' in terms else None,
           'add': add if 'add' in terms else None}
    xs = _place(x, offset)
    G = 64 * C
    y = Guarded((rows, C), BF16, G, offset=offset)
    _call('og_ln_rows_fwd', xs.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-5, y.ptr(), rows, C)
    dx = Guarded((rows, C), BF16, G, offset=offset)
    dg, db = Guarded((C,), F32T, G, dg0), Guarded((C,), F32T, G, db0)
    keep = {n: (None if t is None else _place(t, offset)) for n, t in use.items()}
    g0s = _place(g0, offset)
    _call('og_ln_rows_bwd', xs.data_ptr(), gamma.data_ptr(), 1e-5, g0s.data_ptr(),
          *(None if keep[n] is None else keep[n].data_ptr() for n in ('g1', 'g2', 'add')), dx.ptr(), dg.ptr(),
          db.ptr(), rows, C)
    torch.cuda.synchronize()
    for n, o in (('y', y), ('dx', dx), ('dgamma', dg), ('dbeta', db)):
        o.check_guard(n)
    st = ln_ref(x.double(), gamma, beta)
    g = g0.double() + sum(t.double() for t in (use['g1'], use['g2']) if t is not None)
    a = use['add'].double() if use['add'] is not None else torch.zeros_like(g)
    ex = {**ln_fwd_expect(st, gamma, beta), **rope_ln_bwd_expect(st, g, gamma, a, dg_init=dg0, db_init=db0)}
    check_all({'y': y.t, 'dx': dx.t, 'dgamma': dg.t, 'dbeta': db.t}, ex)


@GPU
@pytest.mark.parametrize('terms', ['g0', 'g0+add', 'g0+g1+g2+add'])
@pytest.mark.parametrize('offset', [0, 2])
@pytest.mark.parametrize('C', [16, 48, 96, 256, 512, 1024])
def test_ln_rows_kernels(C, offset, terms):
    """105 rows (not a multiple of the 8 warps of a block), every width the modules reach and the three vectorised
    ones, aligned and misaligned, with g1 / g2 / add NULL and given, dgamma / dbeta pre-filled."""
    ln_rows_run(105, C, terms, offset, seed=50000 + C + 10 * offset + len(terms))


@GPU
@pytest.mark.parametrize('offset', [0, 2])
@pytest.mark.parametrize('C', [64, 256, 1024])
def test_ln_rows_kernels_many_rows(C, offset):
    """More rows than the capped grids have warps: every warp loops over rows and adds its dgamma / dbeta once."""
    ln_rows_run(20000, C, 'g0+g1+g2+add', offset, seed=51000 + C + offset)


@GPU
@pytest.mark.parametrize('offset,kind', [(0, 'vec'), (2, 'generic')])
def test_ln_rows_kernel_names(offset, kind):
    names = [n for n in _kernels_run(lambda: ln_rows_run(24, 512, 'g0+g1+g2+add', offset, seed=52000)) if 'og_' in n]
    want = (['og_ln_rows_fwd_vec_kernel<2>', 'og_ln_rows_bwd_vec_kernel<2>'] if kind == 'vec' else
            ['og_ln_rows_fwd_kernel(', 'og_ln_rows_bwd_kernel('])
    for w in want:
        assert any(w in n for n in names), (w, sorted(set(names)))
    assert not any('og_rope' in n for n in names), sorted(set(names))
    if kind == 'generic':
        assert not any('_vec_kernel' in n for n in names), sorted(set(names))


# ------------------------------------------------------------------------------------------------------------------
# GPU, module level
# ------------------------------------------------------------------------------------------------------------------
def _grads(m):
    return {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}


def _check_block(m, ref_fn, sd, shape, tag, cond_dim, transpose=False):
    """Forward and backward of the module against the oracle, with the tolerances of the d_head = 16 / 128 tests."""
    x = O.det_uniform(tag + '.x', shape)
    gy = O.det_uniform(tag + '.gy', shape, 1e-3)
    cond = O.det_uniform(tag + '.cond', (shape[0], shape[2 if transpose else 1], cond_dim)).sign() if cond_dim else None
    xr = x.clone().requires_grad_(True)
    ref_sd = _ref_sd(sd)
    yr = ref_fn(identity_embed(ref_sd), xr, cond)
    yr.backward(gy)
    xg = x.to(DEV).requires_grad_(True)
    y = m(xg, cond=(None, cond.to(DEV))) if cond_dim else m(xg)
    y.backward(gy.to(DEV).to(y.dtype))
    assert rel_l2(y.float().cpu(), yr.detach()) < 2e-2
    assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2
    grads = _grads(m)
    assert grads and all(ref_sd[k].grad is not None for k in grads)
    for k, g in grads.items():
        assert rel_l2(g, ref_sd[k].grad) < 8e-2, (k, rel_l2(g, ref_sd[k].grad))


@GPU
@pytest.mark.parametrize('T', [16, 64])
@pytest.mark.parametrize('cond_dim', [None, 4])
@pytest.mark.parametrize('nh,dh', [(4, 16), (2, 64), (1, 128)])
def test_spacetime_block_noembed_against_oracle(nh, dh, cond_dim, T):
    """d_head 16, 64 and 128; T = 16 runs the per-pixel temporal kernels at 64 and T = 64 the tiled ones; key_dim runs
    the broadcast-K/V path."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
    m = SpaceTimeAttention(n_head=nh, d_head=dh, embed=False, transpose=False, **kw)
    sd = det_weights(m)
    m.to(DEV)
    _check_block(m, lambda s, x, c: O.spacetime_attention(s, '', x, nh, False, c), sd, (2, T, 4, 4, nh * dh),
                 f'noembed.st.{nh}.{dh}.{cond_dim}.{T}', cond_dim)


@GPU
@pytest.mark.parametrize('embed', [(False, True), (True, False)], ids=str)
@pytest.mark.parametrize('T', [16, 40])
def test_spacetime_block_mixed_embed_against_oracle(embed, T):
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=2, d_head=64, embed=embed, transpose=False)
    sd = det_weights(m)
    m.to(DEV)
    _check_block(m, lambda s, x, c: O.spacetime_attention(s, '', x, 2, False, c), sd, (2, T, 4, 4, 128),
                 f'noembed.mixed.{embed}.{T}', None)


@GPU
def test_spacetime_block_noembed_ffn_transpose_against_oracle():
    """embed=False with transpose=True, a hidden FFN layer, biases, a key_dim conditioning and d_out != n_head*d_head."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=2, d_head=64, embed=False, transpose=True, hid_dim=192, d_out=64, bias=True,
                           time_attn_kw={'key_dim': 4})
    sd = det_weights(m)
    m.to(DEV)
    x = O.det_uniform('noembed.ffn.x', (2, 128, 6, 4, 4))
    cond = O.det_uniform('noembed.ffn.cond', (2, 6, 4)).sign()
    gy = O.det_uniform('noembed.ffn.gy', (2, 64, 6, 4, 4), 1e-3)
    ref_sd = _ref_sd(sd)
    xr = x.clone().requires_grad_(True)
    yr = ffn_oracle.spacetime_attention(identity_embed(ref_sd), '', xr, 2, True, cond)
    yr.backward(gy)
    xg = x.to(DEV).requires_grad_(True)
    y = m(xg, cond=(None, cond.to(DEV)))
    y.backward(gy.to(DEV).to(y.dtype))
    assert rel_l2(y.float().cpu(), yr.detach()) < 2e-2
    assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2
    for k, g in _grads(m).items():
        assert torch.isfinite(g).all(), k
        if k.endswith('to_k.bias'):
            # a bias on every key adds q.b to all scores of a row, which the softmax cancels: its gradient is zero in
            # exact arithmetic, and what either side computes is rounding noise
            continue
        assert rel_l2(g, ref_sd[k].grad) < 8e-2, (k, rel_l2(g, ref_sd[k].grad))


@GPU
@pytest.mark.parametrize('nh,dh,cond_dim,T', [(4, 16, None, 16), (2, 64, 4, 40)])
def test_spacetime_block_noembed_dropout_against_oracle(nh, dh, cond_dim, T):
    """With dropout: the oracle is fed the masks of the seeds the block drew (test_gpu_attention_dropout's method)."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    from test_gpu_attention_dropout import _values, oracle_with_seeds, recorded_seeds
    p = 0.1
    torch.manual_seed(53000 + T)
    kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
    m = SpaceTimeAttention(n_head=nh, d_head=dh, embed=False, transpose=False, dropout=p, **kw)
    sd = det_weights(m)
    m.to(DEV)
    shape = (2, T, 4, 4, nh * dh)
    tag = f'noembed.drop.{nh}.{dh}.{T}'
    x = O.det_uniform(tag + '.x', shape)
    gy = O.det_uniform(tag + '.gy', shape, 1e-3)
    cond = O.det_uniform(tag + '.cond', (2, T, cond_dim)).sign() if cond_dim else None
    xg = x.to(DEV).requires_grad_(True)
    with recorded_seeds() as seeds:
        y = m(xg, cond=(None, cond.to(DEV))) if cond_dim else m(xg)
    y.backward(gy.to(DEV).to(y.dtype))
    assert len(seeds) == 2
    ref_sd = _ref_sd(sd)
    xr = x.clone().requires_grad_(True)
    with oracle_with_seeds(_values(seeds), p) as left:
        yr = O.spacetime_attention(identity_embed(ref_sd), '', xr, nh, False, cond)
    assert not left
    yr.backward(gy)
    assert rel_l2(y.float().cpu(), yr.detach()) < 2e-2
    assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2
    for k, g in _grads(m).items():
        assert rel_l2(g, ref_sd[k].grad) < 0.1, (k, rel_l2(g, ref_sd[k].grad))
    with oracle_with_seeds([v + 1 for v in _values(seeds)], p):
        y_other = O.spacetime_attention(identity_embed(_ref_sd(sd)), '', x, nh, False, cond)
    assert rel_l2(y.float().cpu(), y_other.detach()) > 2e-2


@GPU
@pytest.mark.parametrize('tag', ATTN_CASES + ST_CASES)
def test_golden_noembed_on_gpu(golden, tag):
    """The modules against the reference's own outputs and gradients: samples within the bf16 model tolerances, every
    gradient norm within 5 %. The stand-alone attentions return attention(x) without the skip: the module computes
    bf16(x + attention(x)) - x, rounded at the magnitude of x, so their outputs get 6e-2 where the blocks get 2e-2."""
    c = golden(GOLDEN)[tag]
    m = _golden_module(c)
    det_weights(m)
    m.to(DEV)
    x, cond = _golden_inputs(tag, c)
    xg = x.to(DEV).requires_grad_(True)
    cd = None if cond is None else cond.to(DEV)
    y = m(xg, cond=cd) if 'cls' in c else (m(xg, cond=(None, cd)) if cd is not None else m(xg))
    y.float().square().mean().backward()
    n = c['y'].numel()
    assert rel_l2(_sample(f'noembed.y.{tag}', y, n), c['y']) < (6e-2 if 'cls' in c else 2e-2)
    assert rel_l2(_sample(f'noembed.dx.{tag}', xg.grad, n), c['dx']) < 6e-2
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads(f'noembed.g.{tag}', c, grads):
        assert rel_l2(got, want) < 0.1, (k, rel_l2(got, want))
        assert abs(grads[k].float().norm().item() - norm) <= 0.05 * norm + 1e-6, k


@GPU
def test_golden_noembed_dynamics_on_gpu(golden):
    """A DynamicsModel whose blueprint passes embed=False: loss, gradients and logits against the reference's."""
    import open_genie_b200 as og
    c = golden(GOLDEN)['dynamics']
    dm = og.DynamicsModel(DYN_DESC, **DYN)
    det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = c['tokens'].to(DEV), c['act'].to(DEV), c['mask'].to(DEV)
    logits, _ = dm(tokens, act)
    assert rel_l2(_sample('noembed.dyn.logits', logits, c['logits'].numel()), c['logits']) < 2e-2
    loss = dm.compute_loss(tokens, act, mask=mask)
    loss.backward()
    assert abs(loss.item() - c['loss']) / c['loss'] < 2e-2
    grads = {k: p.grad for k, p in dm.named_parameters() if p.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads('noembed.dyn.g', c, grads):
        assert rel_l2(got, want) < 0.1, (k, rel_l2(got, want))
        assert abs(grads[k].float().norm().item() - norm) <= 0.05 * norm + 1e-6, k


def _entry_points_called(fn):
    """Names of the C-ABI entry points `fn` calls, in order (_lib.TIMING records every call), and the number of kernels
    the library launched meanwhile."""
    from open_genie_b200 import _lib
    n0, _lib.TIMING = _lib.launch_count(), []
    try:
        fn()
        torch.cuda.synchronize()
        return [t[0] for t in _lib.TIMING], _lib.launch_count() - n0
    finally:
        _lib.TIMING = None


@GPU
@pytest.mark.parametrize('embed', [False, (False, True)], ids=str)
def test_noembed_calls_no_rope_entry_point(embed):
    """embed=False calls the LayerNorm-only passes, one launch each (test_ln_rows_kernel_names pins their kernels),
    and never og_rope_table or og_rope_ln_*; with a rotary temporal attention only that attention calls them."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=2, d_head=64, embed=embed, transpose=False)
    det_weights(m)
    m.to(DEV)
    x = O.det_uniform('noembed.names.x', (1, 8, 4, 4, 128)).to(DEV).requires_grad_(True)

    def run():
        y = m(x)
        y.backward(torch.ones_like(y))
    run()                                  # builds the rotary table of the temporal attention, if it has one
    names, launches = _entry_points_called(run)
    assert launches >= len(names) > 0
    rope = [n for n in names if n.startswith('og_rope')]
    if embed is False:
        assert names.count('og_ln_rows_fwd') == names.count('og_ln_rows_bwd') == 2 and not rope, names
    else:
        assert names.count('og_ln_rows_fwd') == names.count('og_ln_rows_bwd') == 1, names
        assert rope == ['og_rope_ln_fwd', 'og_rope_ln_bwd'], names    # the table is cached on the frequencies


class _BlockStep(torch.nn.Module):
    """A SpaceTimeAttention block without rotary embeddings as a GraphedTrainStep model: loss = mean(block(x) * w)."""

    def __init__(self, T):
        super().__init__()
        from open_genie_b200.module.attention import SpaceTimeAttention
        self.block = SpaceTimeAttention(n_head=4, d_head=16, embed=False, transpose=False)
        self.w = O.det_uniform(f'noembed.graph.w.{T}', (2, T, 4, 4, 64)).to(DEV)

    def training_step(self, batch, batch_idx):
        return (self.block(batch).float() * self.w).mean()


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_graphed_train_step_noembed_matches_eager(T):
    """Replays of the captured training step give the loss and gradients of an eager step."""
    from open_genie_b200.graph import GraphedTrainStep
    from open_genie_b200.optim import FusedAdamW
    model = _BlockStep(T)
    det_weights(model.block)
    model.to(DEV)
    opt = FusedAdamW(model.parameters(), lr=0.0, weight_decay=0.0)   # the step's boundary re-zeroes its arena
    x = O.det_uniform(f'noembed.graph.x.{T}', (2, T, 4, 4, 64)).to(DEV)
    step = GraphedTrainStep(model, opt, x)
    results = []
    for _ in range(2):
        loss = step(x)
        torch.cuda.synchronize()
        results.append((loss.item(), {k: g.clone() for k, g in _grads(model).items()}))
    model.zero_grad(set_to_none=True)
    eager = model.training_step(x, 0)
    eager.backward()
    g_e = _grads(model)
    del step                               # release the captured graph before the next test
    torch.cuda.synchronize()
    for l, g in results:
        assert abs(eager.item() - l) <= 1e-3 * abs(l) + 1e-7, (eager.item(), l)
        assert sorted(g) == sorted(g_e)
        for k in g:
            assert rel_l2(g[k], g_e[k]) < 1e-3, (k, rel_l2(g[k], g_e[k]))


@GPU
def test_latent_action_noembed_with_broadcast_kv():
    """Every space-time block of the mini LatentAction without rotary embeddings; the decoder's temporal attention
    takes K / V from the action codes (the broadcast-K/V path)."""
    import open_genie_b200 as og
    noembed = lambda bp: tuple((n, {**kw, 'embed': False} if n == 'space-time_attn' else kw) for n, kw in bp)
    enc, dec = noembed(fx.MINI_ACT_ENC), noembed(fx.MINI_ACT_DEC)
    la = og.LatentAction(enc, dec, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    assert not any(k.endswith('embed.freq') for k in sd)
    la.to(DEV).train()
    video = O.det_uniform('noembed.action.video', fx.MINI_ACT_VIDEO_SHAPE)
    ref_sd = _ref_sd(sd)
    _, ref_loss, (ref_rec, _), _ = O.latent_action_forward(identity_embed(ref_sd), enc, dec, video,
                                                           fx.MINI_ACT_D_CODEBOOK)
    ref_loss.backward()
    idxs, loss, (rec_loss, _) = la(video.to(DEV))
    loss.backward()
    assert abs(rec_loss.item() - ref_rec.item()) / ref_rec.item() < 3e-2
    for k, g in _grads(la).items():
        assert torch.isfinite(g).all(), k
        if k.startswith(('dec_layers', 'proj_out')):
            n = ref_sd[k].grad.norm().item()
            if n > 1e-6:
                assert abs(g.norm().item() - n) / n < 0.1, (k, g.norm().item(), n)
