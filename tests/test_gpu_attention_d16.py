"""Attention heads of width 16: the d_head = 16 flash kernels (csrc/flash_attn.cu), the tiled temporal kernels at
d_head = 16 (csrc/temporal_attn_long.cu), which ops._TimeAttnFn runs at every clip length at that width, and the
modules built on them (the reference's LatentAction / Dynamics examples use 4 heads of 16).

Kernel level: every output element against the float64 references of test_gpu_attention_paths / test_gpu_temporal_long,
with the same per-element bounds and guarded output buffers. Model level: SpaceTimeAttention, DynamicsModel and
LatentAction with 16-wide heads against the CPU oracle (which takes any head width), with the tolerances of the
d_head = 128 model tests. Reference vectors: tests/golden/attn_d16.pt (oracle/make_golden_d16.py, from the unmodified
reference) pins the oracle on the CPU and the modules on the GPU.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from helpers import det_weights, rel_l2
from oracle import fixtures as fx
from oracle import genie_oracle as O
from test_gpu_attention_paths import (BF16, DEV, F32T, Guarded, _call, _kernels_run, _rand, _tseq, check_all,
                                      flash_expect)
from test_gpu_temporal_long import long_expect

GPU = pytest.mark.gpu
D = 16


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation, module construction, dispatch (no device needed)
# ------------------------------------------------------------------------------------------------------------------
def _lib_and_ptr():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    return lib, ctypes.addressof(buf)


def _flash_fwd(lib, p, S=64, C=256, nh=2):
    return lib.og_flash_attn_fwd(p, p, p, p, None, None, p, 1, S, C, nh, 1.0, None)


def _flash_bwd(lib, p, S=64, C=256, nh=2):
    return lib.og_flash_attn_bwd(p, p, p, p, p, p, p, p, p, p, 1, S, C, nh, 1.0, None)


def _long_fwd(lib, q, p, C=256, nh=2):
    return lib.og_temporal_attn_long_fwd(q, p, p, p, None, None, p, 1, 40, 4, C, nh, 1.0, 0, None)


def _long_bwd(lib, q, p, C=256, nh=2):
    return lib.og_temporal_attn_long_bwd(q, p, p, p, p, p, p, p, p, p, None, None, 1, 40, 4, C, nh, 1.0, 0, None)


def test_width_16_passes_the_width_checks():
    """A 16-wide call (C = 16, 48, 256: one, three and sixteen heads) gets past the head-width check of the flash and
    tiled temporal entry points: it is refused only by the next check (an empty problem for flash, a misaligned
    pointer for the tiled kernels). The per-pixel kernels (T <= 32) keep refusing 16: the tiled kernels run every
    clip at that width."""
    lib, p = _lib_and_ptr()
    for nh in (1, 3, 16):
        for call in (_flash_fwd, _flash_bwd):
            assert call(lib, p, S=0, C=D * nh, nh=nh) == -1
            assert b'empty problem' in lib.og_last_error(), lib.og_last_error()
        for call in (_long_fwd, _long_bwd):
            assert call(lib, p + 1, p, C=D * nh, nh=nh) == -1
            assert b'aligned' in lib.og_last_error(), lib.og_last_error()
    assert lib.og_temporal_attn_fwd(p, p, p, None, p, 1, 8, 4, 4 * D, 4, 1.0, 0, None) == -2
    assert b'd_head=16' in lib.og_last_error()
    assert lib.og_temporal_attn_bwd(p, p, p, p, p, p, p, None, None, 1, 8, 4, 4 * D, 4, 1.0, 0, None) == -2
    assert b'd_head=16' in lib.og_last_error()


@pytest.mark.parametrize('d', [8, 24, 32, 48])
def test_other_narrow_widths_are_still_refused(d):
    lib, p = _lib_and_ptr()
    C = 2 * d
    for call in (_flash_fwd, _flash_bwd):
        assert call(lib, p, C=C) == -1 and b'd_head = 64' in lib.og_last_error()
    for call in (_long_fwd, _long_bwd):
        assert call(lib, p, p, C=C) == -2 and b'd_head=%d' % d in lib.og_last_error()
    if d != 32:     # the per-pixel kernels take 32 and 64
        assert lib.og_temporal_attn_fwd(p, p, p, None, p, 1, 8, 4, C, 2, 1.0, 0, None) == -2
        assert b'd_head=%d' % d in lib.og_last_error()
        assert lib.og_temporal_attn_bwd(p, p, p, p, p, p, p, None, None, 1, 8, 4, C, 2, 1.0, 0, None) == -2
        assert b'd_head=%d' % d in lib.og_last_error()


def test_module_accepts_d_head_16():
    from open_genie_b200.module.attention import SpaceTimeAttention, SpatialAttention, TemporalAttention
    for cls in (SpatialAttention, TemporalAttention):
        for nh in (1, 4, 16):
            m = cls(n_head=nh, d_head=D)
            assert m.d_head == D and m.scale == nh / 4
        for d in (8, 32):
            with pytest.raises(NotImplementedError, match='64 or 128'):
                cls(n_head=4, d_head=d)
    m = SpaceTimeAttention(n_head=(4, 1), d_head=(D, 64))
    assert m.space_attn.d_head == D and m.temp_attn.d_head == 64 and m.ffn[1].net[0].num_groups == 1
    m = SpaceTimeAttention(n_head=16, d_head=D)
    assert m.in_channels == 256 and m.ffn[1].net[0].num_groups == 16


def test_time_attention_dispatch_rule_d16():
    """d_head = 16 runs the tiled kernels at every clip length, as d_head = 128 does; 64 keeps its rule."""
    from open_genie_b200 import ops
    for nh in (1, 4, 16):
        for T in (1, 16, 32, 33, 200):
            assert ops._time_attn_tiled(T, D * nh, nh)
    assert not ops._time_attn_tiled(32, 256, 4) and ops._time_attn_tiled(33, 256, 4)


# ------------------------------------------------------------------------------------------------------------------
# flash attention, kernel level
# ------------------------------------------------------------------------------------------------------------------
def flash16_run(nseq, S, nh, seed, amp=0.5, aliased=False):
    C, scale = D * nh, nh * D ** -0.5
    q = _rand((nseq, S, C), seed, amp)
    k, v = (q, q) if aliased else (_rand((nseq, S, C), seed + 1, amp), _rand((nseq, S, C), seed + 2))
    res, do = _rand((nseq, S, C), seed + 3), _rand((nseq, S, C), seed + 4)
    G = 64 * C
    outs = {n: Guarded(q.shape, BF16, G) for n in ('out', 'out_res', 'dq', 'dk', 'dv')}
    outs['lse'] = Guarded((nseq, nh, S), F32T, G)
    delta = Guarded((nseq, nh, S), F32T, G)
    _call('og_flash_attn_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), res.data_ptr(),
          outs['out_res'].ptr(), outs['lse'].ptr(), nseq, S, C, nh, scale)
    _call('og_flash_attn_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), do.data_ptr(),
          outs['lse'].ptr(), delta.ptr(), outs['dq'].ptr(), outs['dk'].ptr(), outs['dv'].ptr(), nseq, S, C, nh, scale)
    torch.cuda.synchronize()
    check_all({n: o.t for n, o in outs.items()}, flash_expect(q, k, v, do, res, nh, scale))
    for n, o in list(outs.items()) + [('delta', delta)]:
        o.check_guard(n)


@GPU
@pytest.mark.parametrize('nh', [1, 3, 4, 16])
@pytest.mark.parametrize('S', [1, 16, 63, 65, 100, 257])
def test_flash16_ragged_S(S, nh):
    flash16_run(nseq=3, S=S, nh=nh, seed=40000 + 10 * S + nh)


@GPU
def test_flash16_full_size_frame():
    flash16_run(nseq=1, S=4096, nh=4, seed=40500)


@GPU
@pytest.mark.parametrize('S,nh', [(100, 4), (256, 16)])
def test_flash16_aliased_product_call(S, nh):
    flash16_run(nseq=2, S=S, nh=nh, seed=40700 + S, aliased=True)


# ------------------------------------------------------------------------------------------------------------------
# tiled temporal attention, kernel level
# ------------------------------------------------------------------------------------------------------------------
def long16_run(B, T, P, nh, bcast, seed, amp=1.0, aliased=False, do_mask=None, check_guards=True):
    C, scale = D * nh, nh * D ** -0.5
    q = _rand((B, T, P, C), seed, amp)
    if aliased:
        k = v = q
    else:
        kvshape = (B, T, C) if bcast else (B, T, P, C)
        k, v = _rand(kvshape, seed + 1, amp), _rand(kvshape, seed + 2)
    res, do = _rand((B, T, P, C), seed + 3), _rand((B, T, P, C), seed + 4)
    if do_mask is not None:
        do = do * do_mask
    G = 64 * C
    outs = {n: Guarded(q.shape, BF16, G) for n in ('out', 'out_res', 'dq')}
    outs['lse'] = Guarded((B, nh, P, T), F32T, G)
    delta = Guarded((B, nh, P, T), F32T, G)
    _call('og_temporal_attn_long_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), res.data_ptr(),
          outs['out_res'].ptr(), outs['lse'].ptr(), B, T, P, C, nh, scale, int(bcast))
    dk_init = dv_init = None
    if bcast:
        dk_init, dv_init = _rand((B, T, C), seed + 5).float(), _rand((B, T, C), seed + 6).float()
        outs['dk_bcast'] = Guarded((B, T, C), F32T, G, dk_init)
        outs['dv_bcast'] = Guarded((B, T, C), F32T, G, dv_init)
        dks = (None, None, outs['dk_bcast'].ptr(), outs['dv_bcast'].ptr())
    else:
        outs['dk'], outs['dv'] = Guarded(q.shape, BF16, G), Guarded(q.shape, BF16, G)
        dks = (outs['dk'].ptr(), outs['dv'].ptr(), None, None)
    _call('og_temporal_attn_long_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), outs['out'].ptr(), do.data_ptr(),
          outs['lse'].ptr(), delta.ptr(), outs['dq'].ptr(), *dks, B, T, P, C, nh, scale, int(bcast))
    torch.cuda.synchronize()
    check_all({n: o.t for n, o in outs.items()}, long_expect(q, k, v, do, res, nh, scale, bcast, dk_init, dv_init))
    if check_guards:
        for n, o in list(outs.items()) + [('delta', delta)]:
            o.check_guard(n)
    return {'q': q, 'k': k, 'v': v, 'res': res, 'do': do}, {n: o.t for n, o in outs.items()}


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('T', [1, 2, 15, 16, 17, 32, 33, 64, 65, 130, 1024])
def test_long16_kernels(T, bcast):
    long16_run(2, T, 5, 3, bcast, seed=41000 + 10 * T + bcast)


@GPU
@pytest.mark.parametrize('nh', [1, 16])
def test_long16_head_counts(nh):
    long16_run(2, 70, 3, nh, 0, seed=41300 + nh)


@GPU
def test_long16_aliased_product_call():
    long16_run(2, 100, 6, 4, 0, seed=41500, aliased=True)


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_long16_large_scores(bcast):
    """|scale q.k| far beyond 89 in places: the online rescale must keep exp in range from tile to tile."""
    B, T, P, nh = 2, 130, 4, 4
    inp, _ = long16_run(B, T, P, nh, bcast, seed=41600 + bcast, amp=3.5)
    qs = _tseq(inp['q'].float(), nh)
    ks = (inp['k'].float().view(B, T, nh, D).permute(0, 2, 1, 3)[:, None] if bcast else _tseq(inp['k'].float(), nh))
    s = ((nh * D ** -0.5) * (qs @ ks.transpose(-1, -2))).tril()
    assert s.abs().amax().item() > 89, 'scores too small to overflow exp without the max subtraction'


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_long16_T1_is_exact(bcast):
    """One time step: the softmax is exactly 1, so out = v (+ residual, rounded once) and, without broadcast, dv = dout."""
    B, T, P, nh = 2, 1, 9, 4
    inp, got = long16_run(B, T, P, nh, bcast, seed=41700 + bcast)
    v = inp['v']
    vb = v[:, :, None].expand(B, T, P, nh * D) if bcast else v
    assert torch.equal(got['out'], vb)
    assert torch.equal(got['out_res'], (vb.float() + inp['res'].float()).to(BF16))
    if not bcast:
        assert torch.equal(got['dv'], inp['do'])


@GPU
@pytest.mark.parametrize('T,bcast', [(150, 0), (150, 1), (40, 0), (16, 0), (16, 1)])
def test_long16_causality_is_exact(T, bcast):
    """Changing every input row t' > t0 (q, k and v) leaves output rows <= t0 bit-identical: out, out_res and lse."""
    B, P, nh = 2, 6, 4
    C, scale = nh * D, nh * D ** -0.5
    kvshape = (B, T, C) if bcast else (B, T, P, C)
    q, k, v, res = _rand((B, T, P, C), 42000), _rand(kvshape, 42001), _rand(kvshape, 42002), _rand((B, T, P, C), 42003)
    t0 = T // 2 + 3
    q2, k2, v2 = q.clone(), k.clone(), v.clone()
    for t, s in ((q2, 42004), (k2, 42005), (v2, 42006)):
        t[:, t0 + 1:] = _rand(t[:, t0 + 1:].shape, s, 3.0)
    runs = []
    for qq, kk, vv in ((q, k, v), (q2, k2, v2)):
        o, orr = torch.empty_like(q), torch.empty_like(q)
        lse = torch.empty((B, nh, P, T), dtype=F32T, device=DEV)
        _call('og_temporal_attn_long_fwd', qq.data_ptr(), kk.data_ptr(), vv.data_ptr(), o.data_ptr(), res.data_ptr(),
              orr.data_ptr(), lse.data_ptr(), B, T, P, C, nh, scale, bcast)
        runs.append((o, orr, lse))
    torch.cuda.synchronize()
    (o1, r1, l1), (o2, r2, l2) = runs
    assert torch.equal(o1[:, :t0 + 1], o2[:, :t0 + 1])
    assert torch.equal(r1[:, :t0 + 1], r2[:, :t0 + 1])
    assert torch.equal(l1[..., :t0 + 1], l2[..., :t0 + 1])
    assert not torch.equal(o1[:, t0 + 1:], o2[:, t0 + 1:])


@GPU
def test_long16_bcast_gradient_many_pixel_chunks():
    """kv_bcast = 1 at P = 4096: every (b, h) is split into many pixel chunks, each added into dK / dV on its own; a
    second pass has dO non-zero only on the first two and last two pixels, so a lost or misrouted chunk is caught."""
    B, T, P, nh = 2, 40, 4096, 4
    long16_run(B, T, P, nh, 1, seed=42100)
    edge = torch.zeros(P, device=DEV, dtype=BF16)
    edge[[0, 1, P - 2, P - 1]] = 1
    long16_run(B, T, P, nh, 1, seed=42200, do_mask=edge.view(1, 1, P, 1), check_guards=False)


# ------------------------------------------------------------------------------------------------------------------
# which kernels run at d_head = 16
# ------------------------------------------------------------------------------------------------------------------
FLASH16 = ['og_flash_attn_fwd_d16_kernel', 'og_flash_attn_bwd_d16_kernel<0>', 'og_flash_attn_bwd_d16_kernel<1>',
           'og_attn_delta_d16_kernel']
LONG16 = ['og_temporal_attn_long_fwd_kernel<16>', 'og_temporal_attn_long_bwd_dq_kernel<16>',
          'og_temporal_attn_long_bwd_dkdv_kernel<16>']


@GPU
def test_flash16_kernel_names():
    names = [n for n in _kernels_run(lambda: flash16_run(nseq=1, S=65, nh=4, seed=45000)) if 'og_' in n]
    for w in FLASH16:
        assert any(w in n for n in names), (w, sorted(set(names)))
    for a in ('og_flash_attn_fwd_kernel', 'og_flash_attn_bwd_kernel<', 'og_attn_delta_kernel', '_d128_'):
        assert not any(a in n for n in names), (a, sorted(set(names)))


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_time_attention_d16_runs_the_tiled_kernels(T):
    from open_genie_b200 import ops
    B, H, W, nh = 1, 4, 4, 4
    C = D * nh
    x = _rand((B, T, H, W, C), 45100 + T).requires_grad_(True)
    freq = O.rope_freq(C, '1d').to(DEV)
    gamma = torch.ones(C, device=DEV, requires_grad=True)
    beta = torch.zeros(C, device=DEV, requires_grad=True)

    def run():
        y = ops.time_attention_res(x, freq, gamma, beta, nh, nh * D ** -0.5)
        y.backward(torch.ones_like(y))
    names = [n for n in _kernels_run(run) if 'og_' in n]
    for w in LONG16:
        assert any(w in n for n in names), (T, w, sorted(set(names)))
    for a in ('og_temporal_attn_fwd_kernel<', 'og_temporal_attn_bwd_kernel<', '_mma_kernel', '_kernel<64>',
              '_kernel<128>'):
        assert not any(a in n for n in names), (T, a, sorted(set(names)))


# ------------------------------------------------------------------------------------------------------------------
# model level, against the CPU oracle
# ------------------------------------------------------------------------------------------------------------------
def _grads(m):
    return {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}


def _ref_sd(sd):
    return {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith(('freq', 'bit_mask')))
            for k, v in sd.items()}


def _check_block(m, ref_fn, sd, shape, tag, cond_dim, transpose=False):
    x = O.det_uniform(tag + '.x', shape)
    gy = O.det_uniform(tag + '.gy', shape, 1e-3)
    cond = O.det_uniform(tag + '.cond', (shape[0], shape[2 if transpose else 1], cond_dim)).sign() if cond_dim else None
    xr = x.clone().requires_grad_(True)
    ref_sd = _ref_sd(sd)
    yr = ref_fn(ref_sd, xr, cond)
    yr.backward(gy)
    xg = x.to(DEV).requires_grad_(True)
    y = m(xg, cond=(None, cond.to(DEV))) if cond_dim else m(xg)
    y.backward(gy.to(DEV).to(y.dtype))
    assert rel_l2(y.float().cpu(), yr.detach()) < 2e-2
    assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2
    grads = _grads(m)
    ref = {k: ref_sd[k].grad for k in grads}
    assert all(g is not None for g in ref.values())
    for k, g in grads.items():
        assert rel_l2(g, ref[k]) < 8e-2, (k, rel_l2(g, ref[k]))


@GPU
@pytest.mark.parametrize('T', [16, 48])
@pytest.mark.parametrize('cond_dim', [None, 4])
@pytest.mark.parametrize('nh', [4, 16])
def test_spacetime_block_d16_against_oracle(nh, cond_dim, T):
    from open_genie_b200.module.attention import SpaceTimeAttention
    kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
    m = SpaceTimeAttention(n_head=nh, d_head=D, transpose=False, **kw)
    sd = det_weights(m)
    m.to(DEV)
    _check_block(m, lambda s, x, c: O.spacetime_attention(s, '', x, nh, False, c), sd, (2, T, 4, 4, D * nh),
                 f'd16.st.{nh}.{cond_dim}.{T}', cond_dim)


@GPU
@pytest.mark.parametrize('S', [64, 100])
def test_spacetime_block_d16_transposed_frames(S):
    """transpose=True ((B, C, T, H, W) video), frames of 8 x 8 and 10 x 10 tokens (S = 64 and 100)."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    hw = int(S ** 0.5)
    m = SpaceTimeAttention(n_head=4, d_head=D, transpose=True)
    sd = det_weights(m)
    m.to(DEV)
    _check_block(m, lambda s, x, c: O.spacetime_attention(s, '', x, 4, True, c), sd, (2, D * 4, 8, hw, hw),
                 f'd16.st.tr.{S}', None, transpose=True)


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_mixed_width_block_d16_against_oracle(T):
    """Space attention with 4 heads of 16, time attention with 1 head of 64, on the same 64 channels (the FFN's
    GroupNorm takes the temporal head count)."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=(4, 1), d_head=(D, 64), transpose=False)
    sd = det_weights(m)
    m.to(DEV)

    def ref(s, x, cond):
        x = O.spatial_attention(s, 'space_attn.', x, 4, False) + x
        x = O.temporal_attention(s, 'temp_attn.', x, 1, False, cond) + x
        y = F.group_norm(x.movedim(-1, 1), 1, s['ffn.1.net.0.weight'], s['ffn.1.net.0.bias'], 1e-5)
        return F.conv3d(y, s['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x
    _check_block(m, ref, sd, (2, T, 4, 4, 64), f'd16.mixed.{T}', None)


def _dyn_inputs(T, hw, vocab, act_vocab, tag):
    shape = (2, T, hw, hw)
    u = O.det_uniform(f'{tag}.tokens', shape) / (3 ** 0.5)
    tokens = ((u + 1) * 0.5 * vocab).long().clamp(0, vocab - 1)
    ua = O.det_uniform(f'{tag}.act', shape[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * act_vocab).long().clamp(0, act_vocab - 1)
    mask = O.det_uniform(f'{tag}.mask', shape) / (3 ** 0.5) < 0.5
    return tokens, act, mask


# the reference's test/test_dynamics.py configuration (without its n_embd key)
DYN16_DESC = (('space-time_attn', {'n_rep': 4, 'n_head': 4, 'd_head': D, 'transpose': False}),)
DYN16 = dict(tok_vocab=16, act_vocab=4, embed_dim=64)


@GPU
@pytest.mark.parametrize('T,hw', [(10, 16), (40, 8)])
def test_dynamics_d16_against_oracle(T, hw):
    import open_genie_b200 as og
    dm = og.DynamicsModel(DYN16_DESC, **DYN16)
    sd = det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = _dyn_inputs(T, hw, DYN16['tok_vocab'], DYN16['act_vocab'], f'd16.dyn.{T}')
    ref_sd = _ref_sd(sd)
    ref_loss = O.dynamics_loss(ref_sd, DYN16_DESC, tokens, act, mask)
    ref_loss.backward()
    loss = dm.compute_loss(tokens.to(DEV), act.to(DEV), mask=mask.to(DEV))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) / ref_loss.item() < 2e-2
    for k, g in _grads(dm).items():
        r = ref_sd[k].grad
        assert r is not None, k
        assert rel_l2(g, r) < 0.1, (k, rel_l2(g, r))


@GPU
def test_dynamics_d16_trains_and_generates():
    """The test_dynamics.py configuration builds, takes optimiser steps that lower its loss on a fixed batch, and
    samples a next frame."""
    import open_genie_b200 as og
    dm = og.DynamicsModel(DYN16_DESC, **DYN16)
    det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = _dyn_inputs(10, 16, DYN16['tok_vocab'], DYN16['act_vocab'], 'd16.train')
    tokens, act, mask = tokens.to(DEV), act.to(DEV), mask.to(DEV)
    opt = torch.optim.AdamW(dm.parameters(), lr=1e-3)
    losses = []
    for _ in range(8):
        opt.zero_grad(set_to_none=True)
        loss = dm.compute_loss(tokens, act, mask=mask)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0], losses
    dm.eval()
    out = dm.generate(tokens[:, :4], act[:, :4], steps=5)
    assert out.shape == (2, 5, 16, 16) and torch.equal(out[:, :4], tokens[:, :4])
    assert int(out.min()) >= 0 and int(out.max()) < DYN16['tok_vocab']


@GPU
def test_latent_action_d16_against_oracle():
    """Every space-time block with 16-wide heads (8 heads on the blueprints' 128 channels); the decoder's temporal
    attention takes K / V from the action codes (the broadcast-K/V path)."""
    import open_genie_b200 as og
    narrow = lambda bp: tuple((n, {**kw, 'n_head': 8, 'd_head': D} if n == 'space-time_attn' else kw) for n, kw in bp)
    enc, dec = narrow(fx.MINI_ACT_ENC), narrow(fx.MINI_ACT_DEC)
    la = og.LatentAction(enc, dec, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    la.to(DEV).train()
    video = O.det_uniform('d16.action.video', fx.MINI_ACT_VIDEO_SHAPE)
    ref_sd = _ref_sd(sd)
    _, ref_loss, (ref_rec, _), _ = O.latent_action_forward(ref_sd, enc, dec, video, fx.MINI_ACT_D_CODEBOOK)
    ref_loss.backward()
    idxs, loss, (rec_loss, _) = la(video.to(DEV))
    loss.backward()
    assert abs(rec_loss.item() - ref_rec.item()) / ref_rec.item() < 3e-2
    grads = _grads(la)
    for k, g in grads.items():
        assert torch.isfinite(g).all(), k
        if k.startswith(('dec_layers', 'proj_out')):
            n = ref_sd[k].grad.norm().item()
            if n > 1e-6:
                assert abs(g.norm().item() - n) / n < 0.1, (k, g.norm().item(), n)


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_spacetime_block_d16_cuda_graph_replay_matches_eager(T):
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=4, d_head=D, transpose=False)
    det_weights(m)
    m.to(DEV)
    shape = (2, T, 4, 4, 4 * D)
    x = O.det_uniform(f'd16.graph.x.{T}', shape).to(DEV).requires_grad_(True)
    gy = O.det_uniform(f'd16.graph.gy.{T}', shape, 1e-3).to(DEV)

    def step():
        y = m(x)
        y.backward(gy.to(y.dtype))
        return y
    y_e = step().detach().float().clone()
    dx_e, g_e = x.grad.float().clone(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = None
            m.zero_grad(set_to_none=True)
            step()
    torch.cuda.current_stream().wait_stream(s)
    x.grad = None
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_g = step()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_l2(y_g.float().cpu(), y_e.cpu()) < 2e-2
    assert rel_l2(x.grad.float().cpu(), dx_e.cpu()) < 6e-2
    for k, p in m.named_parameters():
        if k in g_e:
            assert rel_l2(p.grad.float().cpu(), g_e[k].float().cpu()) < 8e-2, k


# ------------------------------------------------------------------------------------------------------------------
# reference-pinned vectors (tests/golden/attn_d16.pt, written by oracle/make_golden_d16.py from the unmodified
# reference): the oracle on the CPU, the modules on the GPU
# ------------------------------------------------------------------------------------------------------------------
GOLDEN = 'attn_d16.pt'
ST_CASES = ('h4_t0_s64', 'h4_t0_s100_c4', 'h4_t0_s256', 'h4_t1_s64_c4', 'h4_t1_s100', 'h4_t1_s256_c4', 'h16_t0_s64',
            'mixed_t0_s64')


def _sample(key, t, n):
    """The elements oracle/make_golden_d16.py stored of `t`."""
    return t.detach().float().cpu().flatten()[O.det_indices(key, t.numel(), n)]


def _golden_grads(prefix, c, grads):
    """(name, sample of the gradient, stored sample, stored norm) for every gradient of a golden case."""
    return [(k, _sample(f'{prefix}.{k}', grads[k], 32), c['grad'][k], c['grad_norm'][k]) for k in c['grad_names']]


def _golden_block(c):
    from open_genie_b200.module.attention import SpaceTimeAttention
    kw = {'time_attn_kw': {'key_dim': c['key_dim']}} if c['key_dim'] else {}
    return SpaceTimeAttention(n_head=c['n_head'], d_head=c['d_head'], transpose=c['transpose'], **kw)


def _golden_block_inputs(tag, c):
    shape = c['shape']
    x = O.det_uniform(f'd16.x.{tag}', shape)
    t = shape[2] if c['transpose'] else shape[1]
    cond = O.det_uniform(f'd16.cond.{tag}', (shape[0], t, c['key_dim'])).sign() if c['key_dim'] else None
    return x, cond


def _oracle_block(sd, x, c, cond):
    nh = c['n_head']
    if isinstance(nh, int):
        return O.spacetime_attention(sd, '', x, nh, c['transpose'], cond)
    x = x.movedim(1, -1) if c['transpose'] else x
    x = O.spatial_attention(sd, 'space_attn.', x, nh[0], False) + x
    x = O.temporal_attention(sd, 'temp_attn.', x, nh[1], False, cond) + x
    y = F.group_norm(x.movedim(-1, 1), nh[1], sd['ffn.1.net.0.weight'], sd['ffn.1.net.0.bias'], 1e-5)
    y = F.conv3d(y, sd['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x
    return y.movedim(-1, 1) if c['transpose'] else y


def _narrow(bp):
    return tuple((n, {**kw, 'n_head': 8, 'd_head': D} if n == 'space-time_attn' else kw) for n, kw in bp)


def test_golden_d16_holds_every_case(golden):
    g = golden(GOLDEN)
    assert tuple(g) == ST_CASES + ('dynamics', 'latent_action')
    assert g['dynamics']['desc'] == DYN16_DESC and g['dynamics']['kw'] == DYN16
    assert g['latent_action']['enc'] == _narrow(fx.MINI_ACT_ENC) and g['latent_action']['dec'] == _narrow(fx.MINI_ACT_DEC)


@pytest.mark.parametrize('tag', ST_CASES)
def test_golden_d16_oracle_blocks(golden, tag):
    """The CPU oracle reproduces the reference's blocks with 16-wide heads; the module's state_dict is the
    reference's."""
    c = golden(GOLDEN)[tag]
    m = _golden_block(c)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == c['keys']
    sd = det_weights(m)
    ref = {k: v.clone().requires_grad_(not k.endswith('freq')) for k, v in sd.items()}
    x, cond = _golden_block_inputs(tag, c)
    x.requires_grad_(True)
    y = _oracle_block(ref, x, c, cond)
    y.square().mean().backward()
    n = c['y'].numel()
    torch.testing.assert_close(_sample(f'd16.y.{tag}', y, n), c['y'], rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(_sample(f'd16.dx.{tag}', x.grad, n), c['dx'], rtol=2e-4, atol=1e-6)
    grads = {k: v.grad for k, v in ref.items() if v.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads(f'd16.g.{tag}', c, grads):
        torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-6)
        assert abs(grads[k].norm().item() - norm) <= 1e-4 * norm + 1e-7, k


def test_golden_d16_oracle_dynamics(golden):
    import open_genie_b200 as og
    c = golden(GOLDEN)['dynamics']
    dm = og.DynamicsModel(DYN16_DESC, **DYN16)
    assert {k: tuple(v.shape) for k, v in dm.state_dict().items()} == c['keys']
    sd = det_weights(dm)
    ref = _ref_sd(sd)
    logits = O.dynamics_forward(ref, DYN16_DESC, c['tokens'], c['act'])
    assert tuple(logits.shape) == c['logits_shape']
    torch.testing.assert_close(_sample('d16.dyn.logits', logits, c['logits'].numel()), c['logits'], rtol=2e-4,
                               atol=2e-5)
    loss = O.dynamics_loss(ref, DYN16_DESC, c['tokens'], c['act'], c['mask'])
    loss.backward()
    assert abs(loss.item() - c['loss']) <= 2e-4 * abs(c['loss'])
    grads = {k: v.grad for k, v in ref.items() if v.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads('d16.dyn.g', c, grads):
        torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-6)
        assert abs(grads[k].norm().item() - norm) <= 1e-4 * norm + 1e-7, k


def test_golden_d16_oracle_latent_action(golden):
    c = golden(GOLDEN)['latent_action']
    import open_genie_b200 as og
    la = og.LatentAction(c['enc'], c['dec'], d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    video = O.det_uniform('d16.action.video', fx.MINI_ACT_VIDEO_SHAPE)
    idxs, loss, (rec, _), _ = O.latent_action_forward(sd, c['enc'], c['dec'], video, fx.MINI_ACT_D_CODEBOOK)
    assert torch.equal(idxs, c['idxs'])
    assert abs(loss.item() - c['loss']) <= 2e-4 * abs(c['loss'])
    assert abs(rec.item() - c['rec_loss']) <= 2e-4 * abs(c['rec_loss'])


@GPU
@pytest.mark.parametrize('tag', ST_CASES)
def test_golden_d16_blocks_on_gpu(golden, tag):
    """The modules against the reference's own outputs and gradients: samples within the bf16 model tolerances, every
    gradient norm within 5 %."""
    c = golden(GOLDEN)[tag]
    m = _golden_block(c)
    det_weights(m)
    m.to(DEV)
    x, cond = _golden_block_inputs(tag, c)
    xg = x.to(DEV).requires_grad_(True)
    y = m(xg, cond=(None, cond.to(DEV))) if cond is not None else m(xg)
    y.float().square().mean().backward()
    n = c['y'].numel()
    assert rel_l2(_sample(f'd16.y.{tag}', y, n), c['y']) < 2e-2
    assert rel_l2(_sample(f'd16.dx.{tag}', xg.grad, n), c['dx']) < 6e-2
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads(f'd16.g.{tag}', c, grads):
        assert rel_l2(got, want) < 0.1, (k, rel_l2(got, want))
        assert abs(grads[k].float().norm().item() - norm) <= 0.05 * norm + 1e-6, k


@GPU
def test_golden_d16_dynamics_on_gpu(golden):
    """The reference's test_dynamics.py configuration: loss, gradients and logits against the reference's."""
    import open_genie_b200 as og
    c = golden(GOLDEN)['dynamics']
    dm = og.DynamicsModel(DYN16_DESC, **DYN16)
    det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = c['tokens'].to(DEV), c['act'].to(DEV), c['mask'].to(DEV)
    logits, _ = dm(tokens, act)
    assert rel_l2(_sample('d16.dyn.logits', logits, c['logits'].numel()), c['logits']) < 2e-2
    loss = dm.compute_loss(tokens, act, mask=mask)
    loss.backward()
    assert abs(loss.item() - c['loss']) / c['loss'] < 2e-2
    grads = {k: p.grad for k, p in dm.named_parameters() if p.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads('d16.dyn.g', c, grads):
        assert rel_l2(got, want) < 0.1, (k, rel_l2(got, want))
        assert abs(grads[k].float().norm().item() - norm) <= 0.05 * norm + 1e-6, k
