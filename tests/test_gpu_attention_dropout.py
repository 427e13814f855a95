"""Attention dropout: SDPA's dropout_p in the flash kernels (csrc/flash_attn.cu) and the tiled temporal kernels
(csrc/temporal_attn_long.cu), through og_flash_attn_dropout_fwd / bwd and og_temporal_attn_long_dropout_fwd / bwd,
and the modules built on them (`Attention(dropout=p)`, SpaceTimeAttention, DynamicsModel, LatentAction).

The mask (csrc/attn_dropout.cuh) is restated here in torch integer arithmetic (`philox4x32_10`, `keep_mask`) and
pinned on the CPU to the Random123 known-answer vectors. With it, every kernel output is checked element by element
against float64 within per-element bounds built like test_gpu_attention_paths.attn_err (`drop_err`), in guarded
buffers; the CPU tests show that the bounds reject the plausible dropout mistakes. Model level, the CPU oracle runs
with the masks of the seeds the modules drew (recorded by wrapping ops._dropout_seed).
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from helpers import Guarded, det_weights, rel_l2
from oracle import fixtures as fx
from oracle import genie_oracle as O
from test_gpu_attention_paths import (BF16, DEV, F32T, SLACK, U, _call, _cpu_rand, _kvseq, _kvsum, _rand, _rejects,
                                      _tseq, _tunseq, bf16_tol, check_all, gam)

GPU = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------------------------
# the mask, restated
# ------------------------------------------------------------------------------------------------------------------
M32 = 0xFFFFFFFF
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def philox4x32_10(c, key):
    """Philox4x32-10 (Salmon et al. 2011) on int64 tensors holding uint32 values (broadcast together). A product of
    two uint32 may wrap in int64; its low 64 bits are exact, and the masks below take the two halves."""
    c0, c1, c2, c3 = c
    k0, k1 = key
    for _ in range(10):
        p0, p1 = c0 * PHILOX_M[0], c2 * PHILOX_M[1]
        c0, c1, c2, c3 = ((p1 >> 32) & M32) ^ c1 ^ k0, p1 & M32, ((p0 >> 32) & M32) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + PHILOX_W[0]) & M32, (k1 + PHILOX_W[1]) & M32
    return c0, c1, c2, c3


def f32(p):
    """p as the entry points receive it (a C float)."""
    return torch.tensor(p, dtype=torch.float32).item()


def threshold(p):
    return min(round(f32(p) * 2 ** 32), 2 ** 32 - 1)


def keep_mask(seed, z, nq, nk, p):
    """bool [*z.shape, nq, nk]: keep(i, j) for the sequence-head indices z = sequence * n_head + head (int64 tensor),
    queries i < nq, keys j < nk (csrc/attn_dropout.cuh)."""
    dev = z.device
    i = torch.arange(nq, device=dev).view(nq, 1)
    j = torch.arange(nk, device=dev).view(1, nk)
    zz = z[..., None, None]
    s = seed & (2 ** 64 - 1)
    w = philox4x32_10(((j >> 4) * 8 + (j & 7), (i >> 4) * 8 + (i & 7), zz & M32, (zz >> 32) & M32),
                      (s & M32, s >> 32))
    sel = 2 * ((i >> 3) & 1) + ((j >> 3) & 1)
    word = torch.where(sel == 0, w[0], torch.where(sel == 1, w[1], torch.where(sel == 2, w[2], w[3])))
    return word >= threshold(p)


def _seed_tensor(v, device=DEV):
    """A seed value as the kernels read it: one int64 whose bits are the uint64 seed."""
    v &= 2 ** 64 - 1
    return torch.tensor([v - 2 ** 64 if v >= 2 ** 63 else v], dtype=torch.int64, device=device)


def test_philox_known_answers():
    """The restatement reproduces Random123's known-answer vectors for Philox4x32-10."""
    t = lambda *v: tuple(torch.tensor(x, dtype=torch.int64) for x in v)
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((M32,) * 4, (M32, M32), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for c, k, want in cases:
        got = philox4x32_10(t(*c), tuple(k))
        assert tuple(int(x) for x in got) == want, [hex(int(x)) for x in got]


def test_keep_mask_groups_each_call_on_i_i8_j_j8():
    """One Philox call's four words decide {i, i + 8} x {j, j + 8}: word 2a + b is (i + 8a, j + 8b), and the counter
    does not depend on bit 3 of i or j."""
    seed, z, p = 0x0123456789ABCDEF, 7 * 3 + 2, 0.5
    m = keep_mask(seed, torch.tensor([z]), 64, 64, p)[0]
    s = seed
    for i in (0, 5, 16, 23, 48):
        for j in (0, 3, 16, 39, 50):
            assert (i >> 3) & 1 == 0 and (j >> 3) & 1 == 0
            c = tuple(torch.tensor(x) for x in ((j >> 4) * 8 + (j & 7), (i >> 4) * 8 + (i & 7), z & M32, z >> 32))
            w = philox4x32_10(c, (s & M32, s >> 32))
            for a in (0, 1):
                for b in (0, 1):
                    assert bool(m[i + 8 * a, j + 8 * b]) == (int(w[2 * a + b]) >= threshold(p))
    t = threshold(0.1)
    assert abs((1 - t / 2 ** 32) - (1 - f32(0.1))) <= 2 ** -33
    # sequences, heads and seeds all change the mask; the kept fraction is near 1 - p
    ms = keep_mask(seed, torch.arange(4), 64, 64, 0.3)
    assert all(not torch.equal(ms[a], ms[b]) for a in range(4) for b in range(a))
    assert not torch.equal(ms[0], keep_mask(seed + 1, torch.arange(1), 64, 64, 0.3)[0])
    assert abs(ms.double().mean().item() - 0.7) < 0.02


def test_sdpa_dropout_semantics():
    """What the oracle restates: torch's SDPA with dropout_p multiplies softmax(S * scale) (after the causal mask) by
    M / (1 - p), also under no_grad; causal entries stay zero."""
    S, p = 48, 0.4
    g = torch.Generator().manual_seed(5)
    q, k = torch.randn(1, 2, S, S, generator=g, dtype=torch.float64), torch.randn(1, 2, S, S, generator=g,
                                                                                   dtype=torch.float64)
    v = torch.eye(S, dtype=torch.float64).expand(1, 2, S, S)
    torch.manual_seed(11)
    with torch.no_grad():
        out = F.scaled_dot_product_attention(q, k, v, is_causal=True, dropout_p=p, scale=0.3)
    sm = torch.softmax((0.3 * q @ k.transpose(-1, -2)).masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(),
                                                                     float('-inf')), -1)
    kept = out != 0
    torch.testing.assert_close(out, sm * kept / (1 - p), rtol=1e-12, atol=0)
    assert not kept.triu(1).any()
    frac = kept.tril().double().sum() / (2 * S * (S + 1) / 2)
    assert abs(frac.item() - (1 - p)) < 0.05


# ------------------------------------------------------------------------------------------------------------------
# float64 reference with a mask, and its bounds
# ------------------------------------------------------------------------------------------------------------------
def drop_ref(q, k, v, scale, keep, p, causal=False, do=None, transpose_mask=False, no_rescale=False, dv_undropped=False,
             delta_undropped=False):
    """Explicit attention with dropout on [..., S, d] float64 tensors: P = softmax, P~ = P Z with Z = keep / (1 - p),
    O = P~ V, lse of the undropped scores; dV = P~^T dO, dP = (dO V^T) Z, dS = P (dP - rowsum(dO O)).
    The keyword switches build the mistakes the bounds must reject."""
    s = scale * (q @ k.transpose(-1, -2))
    if causal:
        s = s.masked_fill(~torch.ones(s.shape[-2:], dtype=torch.bool, device=s.device).tril(), float('-inf'))
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    pr = e / l
    kf = keep.transpose(-1, -2) if transpose_mask else keep
    z = kf.double() * (1.0 if no_rescale else 1.0 / (1.0 - f32(p)))
    pt = pr * z
    r = {'p': pr, 'pt': pt, 'z': z, 'o': pt @ v, 'lse': (m + l.log()).squeeze(-1)}
    if do is not None:
        dp = (do @ v.transpose(-1, -2)) * z
        o_delta = pr @ v if delta_undropped else r['o']
        delta = (do * o_delta).sum(-1, keepdim=True)
        ds = pr * (dp - delta)
        r.update(ds=ds, dq=scale * (ds @ k), dk=scale * (ds.transpose(-1, -2) @ q),
                 dv=(pr if dv_undropped else pt).transpose(-1, -2) @ do)
    return r


def drop_err(q, k, v, r, scale, do):
    """attn_err's bound (P and dS rounded to bf16 before their products, delta from the bf16 output) with the mask:
    the products take P~ and |dP Z|; the error of a dropped entry's dS (P times the delta error) keeps P."""
    aq, ak, av = q.abs(), k.abs(), v.abs()
    p, pt, z = r['p'], r['pt'], r['z']
    g = gam(k.shape[-2] + 128)
    es = (gam(2 * q.shape[-1]) * scale) * (aq @ ak.transpose(-1, -2))
    es = torch.where(p > 0, es, torch.zeros_like(es)).amax(-1, keepdim=True)
    rho = g + 2 * es + gam(4) * (1 + r['lse'].abs()).unsqueeze(-1)
    err = {'o': (U + rho) * (pt @ av), 'lse': rho.squeeze(-1)}
    ado = do.abs()
    dp_mag = (ado @ av.transpose(-1, -2)) * z
    ed = (rho + g) * (p * dp_mag).sum(-1, keepdim=True) + (ado * (err['o'] + U * r['o'].abs())).sum(-1, keepdim=True)
    eds = (U + rho + g) * r['ds'].abs() + p * (ed + g * dp_mag)
    err['dq'] = scale * (eds @ ak)
    err['dk'] = scale * (eds.transpose(-1, -2) @ aq)
    err['dv'] = (U + rho + g) * (pt.transpose(-1, -2) @ ado)
    return err


def flash_drop_expect(q, k, v, do, res, nh, scale, keep, p, **mut):
    """{output: (reference, tolerance)} of og_flash_attn_dropout_fwd / bwd on bf16 [nseq, S, C] inputs; keep: bool
    [nseq, nh, S, S]."""
    nseq, S, C = q.shape
    sp = lambda t: t.double().view(nseq, S, nh, C // nh).transpose(1, 2)
    un = lambda t: t.transpose(1, 2).reshape(nseq, S, C)
    qs, ks, vs, dos = sp(q), sp(k), sp(v), sp(do)
    r = drop_ref(qs, ks, vs, scale, keep, p, do=dos, **mut)
    e = drop_err(qs, ks, vs, drop_ref(qs, ks, vs, scale, keep, p, do=dos), scale, dos)
    out = {name: (un(r[name]), bf16_tol(un(e[name]), un(r[name]))) for name in ('o', 'dq', 'dk', 'dv')}
    out['out'] = out.pop('o')
    out['lse'] = (r['lse'], SLACK * e['lse'])
    orr = un(r['o']) + res.double()
    out['out_res'] = (orr, SLACK * (un(e['o']) + U * orr.abs()))
    return out


def long_drop_expect(q, k, v, do, res, nh, scale, bcast, keep, p, dk_init=None, dv_init=None):
    """The same for og_temporal_attn_long_dropout_fwd / bwd: q, do, res [B, T, P, C]; k, v the same or [B, T, C];
    keep: bool [B, P, nh, T, T]."""
    B, T, P, C = q.shape
    f = lambda t: t.double()
    qs, dos = _tseq(f(q), nh), _tseq(f(do), nh)
    ks, vs = (_kvseq(f(k), nh), _kvseq(f(v), nh)) if bcast else (_tseq(f(k), nh), _tseq(f(v), nh))
    r = drop_ref(qs, ks, vs, scale, keep, p, causal=True, do=dos)
    e = drop_err(qs, ks, vs, r, scale, dos)
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


@pytest.mark.parametrize('p', [0.1, 0.5])
def test_tolerances_reject_plausible_dropout_bugs(p):
    """A kernel that is exactly right (the reference rounded to bf16) passes; each dropout mistake is rejected: the
    mask transposed, the 1 / (1 - p) missing, dV taken from the undropped P, delta taken from the undropped O."""
    nseq, S, nh, d = 2, 100, 2, 64
    C, scale = nh * d, nh * d ** -0.5
    q, k, v, do, res = (_cpu_rand((nseq, S, C), 500 + i, 1.0) for i in range(5))
    z = torch.arange(nseq).view(nseq, 1) * nh + torch.arange(nh).view(1, nh)
    keep = keep_mask(0x5EED, z, S, S, p)
    ex = flash_drop_expect(q, k, v, do, res, nh, scale, keep, p)
    exact = {n: (t[0].float() if n == 'lse' else t[0].to(BF16)) for n, t in ex.items()}
    check_all(exact, ex)
    for mut, names in (({'transpose_mask': True}, ('out', 'dq', 'dk', 'dv')),
                       ({'no_rescale': True}, ('out', 'dv')),
                       ({'dv_undropped': True}, ('dv',)),
                       ({'delta_undropped': True}, ('dq', 'dk'))):
        bad = flash_drop_expect(q, k, v, do, res, nh, scale, keep, p, **mut)
        for n in names:
            _rejects({n: bad[n][0].to(BF16)}, ex)
    # and the undropped attention itself
    ex0 = flash_drop_expect(q, k, v, do, res, nh, scale, torch.ones_like(keep), 0.0)
    _rejects({'out': ex0['out'][0].to(BF16)}, ex)


# ------------------------------------------------------------------------------------------------------------------
# CPU: entry points, modules, dispatch
# ------------------------------------------------------------------------------------------------------------------
def _lib_and_ptr():
    import ctypes
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    return lib, ctypes.addressof(buf)


def test_dropout_entry_points_validate_p_and_seed():
    lib, ptr = _lib_and_ptr()
    calls = {
        'flash_fwd': lambda p, sd, S=64, C=256: lib.og_flash_attn_dropout_fwd(ptr, ptr, ptr, ptr, None, None, ptr, 1, S,
                                                                             C, 4, 1.0, p, sd, None),
        'flash_bwd': lambda p, sd, S=64, C=256: lib.og_flash_attn_dropout_bwd(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr,
                                                                             ptr, ptr, 1, S, C, 4, 1.0, p, sd, None),
        'long_fwd': lambda p, sd, S=40, C=256: lib.og_temporal_attn_long_dropout_fwd(
            ptr + 1, ptr, ptr, ptr, None, None, ptr, 1, S, 4, C, 4, 1.0, 0, p, sd, None),
        'long_bwd': lambda p, sd, S=40, C=256: lib.og_temporal_attn_long_dropout_bwd(
            ptr + 1, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, None, 1, S, 4, C, 4, 1.0, 0, p, sd, None),
    }
    for name, call in calls.items():
        assert call(0.1, None) == -1 and b'null seed' in lib.og_last_error(), name
        for p in (-0.1, 1.0, 1.5, float('nan')):
            assert call(p, ptr) == -1 and b'[0, 1)' in lib.og_last_error(), (name, p)
    # otherwise the counterparts' checks, codes and messages
    assert calls['flash_fwd'](0.1, ptr, S=0) == -1 and b'flash_attn_fwd: empty problem' in lib.og_last_error()
    assert calls['flash_bwd'](0.1, ptr, C=96) == -1 and b'flash_attn_bwd: needs d_head' in lib.og_last_error()
    assert calls['long_fwd'](0.1, ptr) == -1 and b'temporal_attn_long_fwd: q, k' in lib.og_last_error()
    assert calls['long_bwd'](0.1, ptr, C=96) == -2 and b'temporal_attn_long_bwd: d_head=24' in lib.og_last_error()


def test_modules_accept_dropout_in_0_1():
    from open_genie_b200.module.attention import SpaceTimeAttention, SpatialAttention, TemporalAttention
    for cls in (SpatialAttention, TemporalAttention):
        for p in (0.0, 0.1, 0.5, 0.999):
            assert cls(n_head=4, d_head=64, dropout=p).dropout == p
        for p in (-0.1, 1.0, 2.0):
            with pytest.raises(NotImplementedError, match=r'\[0, 1\)'):
                cls(n_head=4, d_head=64, dropout=p)
    m = SpaceTimeAttention(n_head=4, d_head=16, dropout=0.1)
    assert m.space_attn.dropout == m.temp_attn.dropout == 0.1
    ref_keys = SpaceTimeAttention(n_head=4, d_head=16).state_dict().keys()
    assert m.state_dict().keys() == ref_keys


def test_blueprints_pass_dropout():
    import open_genie_b200 as og
    desc = (('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 16, 'dropout': 0.1, 'transpose': False}),)
    dm = og.DynamicsModel(desc, tok_vocab=16, act_vocab=4, embed_dim=64)
    drops = [mod.dropout for mod in dm.modules() if hasattr(mod, 'dropout') and hasattr(mod, 'n_head')]
    assert drops and all(p == 0.1 for p in drops)


def test_time_attention_dispatch_rule_with_dropout():
    from open_genie_b200 import ops
    for T in (1, 2, 16, 32, 33, 1024):
        for C, nh in ((256, 4), (64, 4), (512, 4)):
            assert ops._time_attn_tiled(T, C, nh, dropout=0.1)
            assert ops._time_attn_tiled(T, C, nh, dropout=0.0) == ops._time_attn_tiled(T, C, nh)
    assert not ops._time_attn_tiled(32, 256, 4, dropout=0.0) and ops._time_attn_tiled(33, 256, 4, dropout=0.0)


# ------------------------------------------------------------------------------------------------------------------
# the oracle with masks
# ------------------------------------------------------------------------------------------------------------------
def attention_core_keep(sd, pre, x, n_head, causal, kind, cond=None, keep=None, p=0.0):
    """genie_oracle.attention_core with SDPA's dropout made explicit: softmax(S * scale) * keep / (1 - p) @ V in the
    caller's dtype, keep: bool (n, h, q, k). keep=None is genie_oracle.attention_core itself."""
    if keep is None:
        return O.attention_core(sd, pre, x, n_head, causal, kind, cond)
    c = x.shape[-1]
    d_head = c // n_head
    q = O.rope(x, sd[pre + 'embed.freq'])
    q = F.layer_norm(q, (c,), sd[pre + 'norm.weight'], sd[pre + 'norm.bias'], 1e-5)
    if cond is None:
        k = v = q
    else:
        k = F.linear(cond, sd[pre + 'to_qkv.to_k.weight'])
        v = F.linear(cond, sd[pre + 'to_qkv.to_v.weight'])
    split = lambda t: t.reshape(t.shape[0], t.shape[1], n_head, d_head).transpose(1, 2)
    s = (n_head * d_head ** -0.5) * (split(q) @ split(k).transpose(-1, -2))
    if causal:
        s = s.masked_fill(~torch.ones(s.shape[-2:], dtype=torch.bool).tril(), float('-inf'))
    a = torch.softmax(s, -1) * keep.to(s.dtype) / (1 - p)
    o = a @ split(v)
    return o.transpose(1, 2).reshape(x.shape[0], x.shape[1], c)


@contextlib.contextmanager
def oracle_with_seeds(seeds, p):
    """Within the block genie_oracle runs every attention call with the mask of the next recorded seed (the order in
    which the modules drew them: per block, spatial then temporal)."""
    queue = list(seeds)
    core = O.attention_core

    def with_mask(sd, pre, x, n_head, causal, kind, cond=None):
        n, S = x.shape[0], x.shape[1]
        z = torch.arange(n).view(n, 1) * n_head + torch.arange(n_head).view(1, n_head)
        keep = keep_mask(queue.pop(0), z, S, S, p)
        return attention_core_keep(sd, pre, x, n_head, causal, kind, cond, keep, p)
    O.attention_core = with_mask
    try:
        yield queue
    finally:
        O.attention_core = core


@contextlib.contextmanager
def recorded_seeds(replay=None):
    """Wraps ops._dropout_seed: records the seed tensors drawn, or (replay) hands out the given seed values in order."""
    from open_genie_b200 import ops
    drawn, draw = [], ops._dropout_seed
    queue = list(replay or ())

    def wrapped(device):
        t = _seed_tensor(queue.pop(0), device) if replay is not None else draw(device)
        drawn.append(t)
        return t
    ops._dropout_seed = wrapped
    try:
        yield drawn
    finally:
        ops._dropout_seed = draw


def _values(seeds):
    return [int(t.item()) & (2 ** 64 - 1) for t in seeds]


def test_oracle_keep_all_ones_matches_oracle():
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=4, d_head=16, transpose=False)
    sd = det_weights(m)
    x = O.det_uniform('drop.oracle.x', (2, 6, 4, 4, 64))
    for pre, causal, kind in (('space_attn.', False, '2d'), ('temp_attn.', True, '1d')):
        rows = x.reshape(-1, 16, 64) if not causal else x.permute(0, 2, 3, 1, 4).reshape(-1, 6, 64)
        ref = O.attention_core(sd, pre, rows, 4, causal, kind)
        assert torch.equal(attention_core_keep(sd, pre, rows, 4, causal, kind), ref)
        ones = torch.ones(rows.shape[0], 4, rows.shape[1], rows.shape[1], dtype=torch.bool)
        torch.testing.assert_close(attention_core_keep(sd, pre, rows, 4, causal, kind, keep=ones), ref, rtol=2e-6,
                                   atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------
# kernel level: flash attention
# ------------------------------------------------------------------------------------------------------------------
def flash_drop_run(nseq, S, nh, d, p, seed, amp=0.5, aliased=False):
    C, scale = d * nh, nh * d ** -0.5
    q = _rand((nseq, S, C), seed, amp)
    k, v = (q, q) if aliased else (_rand((nseq, S, C), seed + 1, amp), _rand((nseq, S, C), seed + 2))
    res, do = _rand((nseq, S, C), seed + 3), _rand((nseq, S, C), seed + 4)
    G = 64 * C
    outs = {n: Guarded(q.shape, BF16, G) for n in ('out', 'out_res', 'dq', 'dk', 'dv')}
    outs['lse'] = Guarded((nseq, nh, S), F32T, G)
    delta = Guarded((nseq, nh, S), F32T, G)
    sv = (seed * 0x9E3779B97F4A7C15 + 1) & (2 ** 64 - 1)
    sd = _seed_tensor(sv)
    _call('og_flash_attn_dropout_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), res.data_ptr(),
          outs['out_res'].ptr(), outs['lse'].ptr(), nseq, S, C, nh, scale, p, sd.data_ptr())
    _call('og_flash_attn_dropout_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), do.data_ptr(),
          outs['lse'].ptr(), delta.ptr(), outs['dq'].ptr(), outs['dk'].ptr(), outs['dv'].ptr(), nseq, S, C, nh, scale,
          p, sd.data_ptr())
    torch.cuda.synchronize()
    z = torch.arange(nseq, device=DEV).view(nseq, 1) * nh + torch.arange(nh, device=DEV).view(1, nh)
    keep = keep_mask(sv, z, S, S, p)
    check_all({n: o.t for n, o in outs.items()}, flash_drop_expect(q, k, v, do, res, nh, scale, keep, p))
    for n, o in list(outs.items()) + [('delta', delta)]:
        o.check_guard(n)
    return {n: o.t.clone() for n, o in outs.items()}


FLASH_S = [1, 63, 64, 65, 200, 1024, 4096]
PS = [0.1, 0.5, 0.9]


@GPU
@pytest.mark.parametrize('S', FLASH_S)
@pytest.mark.parametrize('d', [16, 64, 128])
def test_flash_dropout_kernels(d, S):
    nh = {1: 16, 63: 3, 64: 1, 65: 4, 200: 2, 1024: 2, 4096: 1}[S]
    nseq = 3 if S <= 200 else 1
    p = PS[(FLASH_S.index(S) + d) % 3]
    flash_drop_run(nseq, S, nh, d, p, seed=60000 + 10 * S + d)


@GPU
@pytest.mark.parametrize('p', PS)
@pytest.mark.parametrize('d', [16, 64, 128])
def test_flash_dropout_aliased_product_call(d, p):
    flash_drop_run(2, 130, 4, d, p, seed=61000 + d, aliased=True)


@GPU
def test_flash_dropout_same_seed_is_bit_identical():
    a = flash_drop_run(2, 200, 4, 64, 0.3, seed=62000)
    b = flash_drop_run(2, 200, 4, 64, 0.3, seed=62000)
    for n in a:
        assert torch.equal(a[n], b[n]), n


# ------------------------------------------------------------------------------------------------------------------
# kernel level: tiled temporal attention
# ------------------------------------------------------------------------------------------------------------------
def long_drop_run(B, T, P, nh, d, bcast, p, seed, amp=1.0):
    C, scale = d * nh, nh * d ** -0.5
    q = _rand((B, T, P, C), seed, amp)
    kvshape = (B, T, C) if bcast else (B, T, P, C)
    k, v = _rand(kvshape, seed + 1, amp), _rand(kvshape, seed + 2)
    res, do = _rand((B, T, P, C), seed + 3), _rand((B, T, P, C), seed + 4)
    G = 64 * C
    outs = {n: Guarded(q.shape, BF16, G) for n in ('out', 'out_res', 'dq')}
    outs['lse'] = Guarded((B, nh, P, T), F32T, G)
    delta = Guarded((B, nh, P, T), F32T, G)
    sv = (seed * 0xD1B54A32D192ED03 + 7) & (2 ** 64 - 1)
    sd = _seed_tensor(sv)
    _call('og_temporal_attn_long_dropout_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(),
          res.data_ptr(), outs['out_res'].ptr(), outs['lse'].ptr(), B, T, P, C, nh, scale, int(bcast), p,
          sd.data_ptr())
    dk_init = dv_init = None
    if bcast:
        dk_init, dv_init = _rand((B, T, C), seed + 5).float(), _rand((B, T, C), seed + 6).float()
        outs['dk_bcast'] = Guarded((B, T, C), F32T, G, dk_init)
        outs['dv_bcast'] = Guarded((B, T, C), F32T, G, dv_init)
        dks = (None, None, outs['dk_bcast'].ptr(), outs['dv_bcast'].ptr())
    else:
        outs['dk'], outs['dv'] = Guarded(q.shape, BF16, G), Guarded(q.shape, BF16, G)
        dks = (outs['dk'].ptr(), outs['dv'].ptr(), None, None)
    _call('og_temporal_attn_long_dropout_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(),
          do.data_ptr(), outs['lse'].ptr(), delta.ptr(), outs['dq'].ptr(), *dks, B, T, P, C, nh, scale, int(bcast), p,
          sd.data_ptr())
    torch.cuda.synchronize()
    z = ((torch.arange(B, device=DEV).view(B, 1, 1) * P + torch.arange(P, device=DEV).view(1, P, 1)) * nh
         + torch.arange(nh, device=DEV).view(1, 1, nh))
    keep = keep_mask(sv, z, T, T, p)
    check_all({n: o.t for n, o in outs.items()},
              long_drop_expect(q, k, v, do, res, nh, scale, bcast, keep, p, dk_init, dv_init))
    for n, o in list(outs.items()) + [('delta', delta)]:
        o.check_guard(n)
    return {n: o.t.clone() for n, o in outs.items()}


LONG_T = [1, 2, 16, 17, 64, 65, 1024]


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('T', LONG_T)
@pytest.mark.parametrize('d', [16, 64, 128])
def test_long_dropout_kernels(d, T, bcast):
    P = 2 if T >= 1024 else 5
    nh = {16: 3, 64: 2, 128: 1}[d]
    p = PS[(LONG_T.index(T) + bcast + d) % 3]
    long_drop_run(2, T, P, nh, d, bcast, p, seed=63000 + 10 * T + d + bcast)


@GPU
def test_long_dropout_same_seed_is_bit_identical():
    a = long_drop_run(2, 100, 4, 4, 64, 0, 0.3, seed=64000)
    b = long_drop_run(2, 100, 4, 4, 64, 0, 0.3, seed=64000)
    for n in a:
        assert torch.equal(a[n], b[n]), n


# ------------------------------------------------------------------------------------------------------------------
# the mask the kernels apply, read back exactly; its statistics
# ------------------------------------------------------------------------------------------------------------------
def _flash_mask_readback(nseq, nh, p, sv):
    """With q = k = 0 every probability of a 64-token frame is 1/64; with V = the identity (d = 64) the output is
    keep(i, j) / (64 (1 - p)), so its non-zero pattern is the kernel's mask. Returns bool [nseq, nh, 64, 64]."""
    S, d = 64, 64
    C = nh * d
    q = torch.zeros((nseq, S, C), dtype=BF16, device=DEV)
    v = torch.eye(S, dtype=BF16, device=DEV).repeat(1, nh).expand(nseq, S, C).contiguous()
    out = torch.empty_like(q)
    lse = torch.empty((nseq, nh, S), dtype=F32T, device=DEV)
    sd = _seed_tensor(sv)
    _call('og_flash_attn_dropout_fwd', q.data_ptr(), q.data_ptr(), v.data_ptr(), out.data_ptr(), None, None,
          lse.data_ptr(), nseq, S, C, nh, 1.0, p, sd.data_ptr())
    torch.cuda.synchronize()
    return (out.view(nseq, S, nh, d).transpose(1, 2) != 0)


@GPU
def test_flash_mask_statistics_and_layout():
    """Over 256 frames x 16 heads x 64 x 64 = 16.8 M scores the kernel's mask equals the restated one bit for bit, its
    kept fraction lies within 5 sigma of 1 - t / 2^32, and different seeds, heads and frames give different masks."""
    nseq, nh, p, sv = 256, 16, 0.1, 0x243F6A8885A308D3
    got = _flash_mask_readback(nseq, nh, p, sv)
    z = torch.arange(nseq, device=DEV).view(nseq, 1) * nh + torch.arange(nh, device=DEV).view(1, nh)
    assert torch.equal(got, keep_mask(sv, z, 64, 64, p))
    n = got.numel()
    q = 1 - threshold(p) / 2 ** 32
    frac = got.double().mean().item()
    assert abs(frac - q) <= 5 * (q * (1 - q) / n) ** 0.5, (frac, q)
    assert not torch.equal(got[0, 0], got[0, 1]) and not torch.equal(got[0, 0], got[1, 0])
    other = _flash_mask_readback(2, 2, p, sv + 1)
    assert not torch.equal(other[0, 0], got[0, 0])


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_long_mask_layout(bcast):
    """The tiled temporal kernels' mask read back exactly (q = k = 0: probability 1 / (t + 1) for keys t' <= t, V = the
    identity), with sequences b * P + p; with broadcast K / V the mask still depends on the pixel."""
    B, T, P, nh, d, p, sv = 2, 64, 3, 2, 64, 0.5, 0x13198A2E03707344
    C = nh * d
    q = torch.zeros((B, T, P, C), dtype=BF16, device=DEV)
    eye = torch.eye(T, dtype=BF16, device=DEV).repeat(1, nh)
    v = (eye.expand(B, T, C) if bcast else eye[:, None].expand(B, T, P, C)).contiguous()
    k = torch.zeros_like(v)
    out = torch.empty_like(q)
    lse = torch.empty((B, nh, P, T), dtype=F32T, device=DEV)
    sd = _seed_tensor(sv)
    _call('og_temporal_attn_long_dropout_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), None, None,
          lse.data_ptr(), B, T, P, C, nh, 1.0, bcast, p, sd.data_ptr())
    torch.cuda.synchronize()
    got = _tseq(out, nh) != 0                      # [B, P, nh, T, T]
    z = ((torch.arange(B, device=DEV).view(B, 1, 1) * P + torch.arange(P, device=DEV).view(1, P, 1)) * nh
         + torch.arange(nh, device=DEV).view(1, 1, nh))
    want = keep_mask(sv, z, T, T, p) & torch.ones(T, T, dtype=torch.bool, device=DEV).tril()
    assert torch.equal(got, want)
    assert not torch.equal(got[0, 0], got[0, 1])


# ------------------------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------------------------
def _grads(m):
    return {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}


def _ref_sd(sd):
    return {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith(('freq', 'bit_mask')))
            for k, v in sd.items()}


def _block_ref(nh, cond):
    if isinstance(nh, int):
        return lambda s, x: O.spacetime_attention(s, '', x, nh, False, cond)

    def ref(s, x):
        x = O.spatial_attention(s, 'space_attn.', x, nh[0], False) + x
        x = O.temporal_attention(s, 'temp_attn.', x, nh[1], False, cond) + x
        y = F.group_norm(x.movedim(-1, 1), nh[1], s['ffn.1.net.0.weight'], s['ffn.1.net.0.bias'], 1e-5)
        return F.conv3d(y, s['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x
    return ref


@GPU
@pytest.mark.parametrize('nh,dh,cond_dim,T', [(4, 16, None, 16), (16, 16, 4, 40), (4, 64, None, 16), (2, 64, 4, 40),
                                              (2, 128, None, 16), ((4, 1), (16, 64), None, 16)])
def test_spacetime_block_dropout_against_oracle(nh, dh, cond_dim, T):
    """Forward and every parameter gradient against the oracle fed the masks of the seeds the block drew (gradients
    within 10 %, the DynamicsModel bound of the d_head = 16 tests: with 16-wide heads the LayerNorm weight gradients
    of the dropped attention are sums of few, noisy terms)."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    p = 0.1
    torch.manual_seed(70000)
    kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
    m = SpaceTimeAttention(n_head=nh, d_head=dh, transpose=False, dropout=p, **kw)
    sd = det_weights(m)
    m.to(DEV)
    C = (nh[1] * dh[1]) if isinstance(nh, tuple) else nh * dh
    shape = (2, T, 4, 4, C)
    tag = f'drop.st.{nh}.{dh}.{cond_dim}.{T}'
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
        yr = _block_ref(nh, cond)(ref_sd, xr)
    assert not left
    yr.backward(gy)
    assert rel_l2(y.float().cpu(), yr.detach()) < 2e-2
    assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2
    for k, g in _grads(m).items():
        assert rel_l2(g, ref_sd[k].grad) < 0.1, (k, rel_l2(g, ref_sd[k].grad))
    # a different mask is far outside these bounds
    with oracle_with_seeds([v + 1 for v in _values(seeds)], p):
        y_other = _block_ref(nh, cond)(_ref_sd(sd), x)
    assert rel_l2(y.float().cpu(), y_other.detach()) > 2e-2


DYN_DESC = (('space-time_attn', {'n_rep': 2, 'n_head': 4, 'd_head': 16, 'dropout': 0.1, 'transpose': False}),)
DYN = dict(tok_vocab=16, act_vocab=4, embed_dim=64)


def _dyn_inputs(T, hw, tag):
    shape = (2, T, hw, hw)
    u = O.det_uniform(f'{tag}.tokens', shape) / (3 ** 0.5)
    tokens = ((u + 1) * 0.5 * DYN['tok_vocab']).long().clamp(0, DYN['tok_vocab'] - 1)
    ua = O.det_uniform(f'{tag}.act', shape[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * DYN['act_vocab']).long().clamp(0, DYN['act_vocab'] - 1)
    mask = O.det_uniform(f'{tag}.mask', shape) / (3 ** 0.5) < 0.5
    return tokens, act, mask


@GPU
def test_dynamics_dropout_loss_and_gradients_against_oracle():
    import open_genie_b200 as og
    dm = og.DynamicsModel(DYN_DESC, **DYN)
    sd = det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = _dyn_inputs(10, 8, 'drop.dyn')
    torch.manual_seed(70100)
    with recorded_seeds() as seeds:
        loss = dm.compute_loss(tokens.to(DEV), act.to(DEV), mask=mask.to(DEV))
    loss.backward()
    assert len(seeds) == 4
    ref_sd = _ref_sd(sd)
    with oracle_with_seeds(_values(seeds), 0.1) as left:
        ref_loss = O.dynamics_loss(ref_sd, DYN_DESC, tokens, act, mask)
    assert not left
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) / ref_loss.item() < 2e-2
    for k, g in _grads(dm).items():
        assert rel_l2(g, ref_sd[k].grad) < 0.1, (k, rel_l2(g, ref_sd[k].grad))


@GPU
def test_dynamics_dropout_drops_in_eval_too():
    """As in the reference (functional SDPA), eval mode and no_grad still drop: the logits and `generate` follow the
    generator's seed; with every attention's dropout set to 0 the logits are deterministic."""
    import open_genie_b200 as og
    dm = og.DynamicsModel(DYN_DESC, **DYN)
    det_weights(dm)
    dm.to(DEV).eval()
    tokens, act, _ = _dyn_inputs(6, 8, 'drop.gen')
    tokens, act = tokens.to(DEV), act.to(DEV)

    def logits(seed):
        torch.manual_seed(seed)
        with torch.no_grad():
            return dm(tokens, act)[0].float()

    def gen(seed):
        torch.manual_seed(seed)
        return dm.generate(tokens[:, :4], act[:, :4], steps=3)
    assert torch.equal(logits(1), logits(1)) and not torch.equal(logits(1), logits(2))
    g1, g2 = gen(3), gen(4)
    assert torch.equal(g1, gen(3)) and not torch.equal(g1, g2)
    for mod in dm.modules():
        if hasattr(mod, 'dropout') and hasattr(mod, 'n_head'):
            mod.dropout = 0.0
    assert torch.equal(logits(1), logits(2))


@GPU
def test_latent_action_dropout_with_broadcast_kv():
    """Every space-time block drops; the decoder's temporal attention takes K / V from the action codes (the
    broadcast-K/V path), against the oracle fed the recorded seeds."""
    import open_genie_b200 as og
    drop = lambda bp: tuple((n, {**kw, 'dropout': 0.1} if n == 'space-time_attn' else kw) for n, kw in bp)
    enc, dec = drop(fx.MINI_ACT_ENC), drop(fx.MINI_ACT_DEC)
    la = og.LatentAction(enc, dec, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    la.to(DEV).train()
    video = O.det_uniform('drop.action.video', fx.MINI_ACT_VIDEO_SHAPE)
    torch.manual_seed(70200)
    with recorded_seeds() as seeds:
        idxs, loss, (rec_loss, _) = la(video.to(DEV))
    loss.backward()
    assert seeds
    ref_sd = _ref_sd(sd)
    with oracle_with_seeds(_values(seeds), 0.1) as left:
        _, ref_loss, (ref_rec, _), _ = O.latent_action_forward(ref_sd, enc, dec, video, fx.MINI_ACT_D_CODEBOOK)
    assert not left
    ref_loss.backward()
    assert abs(rec_loss.item() - ref_rec.item()) / ref_rec.item() < 3e-2
    for k, g in _grads(la).items():
        assert torch.isfinite(g).all(), k
        if k.startswith(('dec_layers', 'proj_out')):
            n = ref_sd[k].grad.norm().item()
            if n > 1e-6:
                assert abs(g.norm().item() - n) / n < 0.1, (k, g.norm().item(), n)


class _BlockStep(torch.nn.Module):
    """A SpaceTimeAttention block with dropout as a GraphedTrainStep model: loss = mean(block(x) * w)."""

    def __init__(self, T):
        super().__init__()
        from open_genie_b200.module.attention import SpaceTimeAttention
        self.block = SpaceTimeAttention(n_head=4, d_head=16, transpose=False, dropout=0.1)
        self.w = O.det_uniform(f'drop.graph.w.{T}', (2, T, 4, 4, 64)).to(DEV)

    def training_step(self, batch, batch_idx):
        return (self.block(batch).float() * self.w).mean()


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_graphed_train_step_draws_fresh_masks(T):
    """Each replay of a captured training step draws new seeds, so new masks; a replay equals an eager step run with
    the seeds that replay drew."""
    from open_genie_b200.graph import GraphedTrainStep
    from open_genie_b200.optim import FusedAdamW
    model = _BlockStep(T)
    det_weights(model.block)
    model.to(DEV)
    opt = FusedAdamW(model.parameters(), lr=0.0, weight_decay=0.0)   # the step's boundary re-zeroes its arena
    x = O.det_uniform(f'drop.graph.x.{T}', (2, T, 4, 4, 64)).to(DEV)
    torch.manual_seed(70300 + T)
    with recorded_seeds() as seeds:
        step = GraphedTrainStep(model, opt, x)
    graph_seeds = seeds[-2:]                       # the captured step's two seed tensors
    results = []
    for _ in range(2):
        loss = step(x)
        torch.cuda.synchronize()
        results.append((_values(graph_seeds), loss.item(), {k: g.clone() for k, g in _grads(model).items()}))
    (s1, l1, g1), (s2, l2, g2) = results
    assert s1 != s2 and l1 != l2
    model.zero_grad(set_to_none=True)
    with recorded_seeds(replay=s2):
        eager = model.training_step(x, 0)
        eager.backward()
    assert abs(eager.item() - l2) <= 1e-3 * abs(l2) + 1e-7
    for k, g in _grads(model).items():
        assert rel_l2(g, g2[k]) < 1e-3, (k, rel_l2(g, g2[k]))
    for k in ('block.space_attn.norm.weight', 'block.temp_attn.norm.weight'):   # the FFN's do not see the masks
        assert rel_l2(g1[k], g2[k]) > 1e-2, k
