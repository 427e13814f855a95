"""Attention heads of width 128: the d_head = 128 flash kernels (csrc/flash_attn.cu), the tiled temporal kernels at
d_head = 128 (csrc/temporal_attn_long.cu), the dispatch of ops._TimeAttnFn at that width, and the modules built on them.

Kernel level: every output element against the float64 references of test_gpu_attention_paths / test_gpu_temporal_long,
with the same per-element bounds and guarded output buffers. Model level: SpaceTimeAttention, DynamicsModel and
LatentAction with 128-wide heads against the CPU oracle (which takes any head width), with the tolerances of the
T > 32 oracle tests.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from helpers import det_weights, rel_l2
from oracle import fixtures as fx
from oracle import genie_oracle as O
from test_gpu_attention_paths import (BF16, DEV, F32T, Guarded, _call, _kernels_run, _kvseq, _rand, _tseq, check_all,
                                      flash_expect)
from test_gpu_temporal_long import long_expect

GPU = pytest.mark.gpu
D = 128


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation (no device needed)
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


def test_width_128_passes_the_width_checks():
    """A 128-wide call gets past the head-width check of all four entry points: it is refused only by the next check
    (an empty problem for flash, a misaligned pointer for the tiled kernels)."""
    lib, p = _lib_and_ptr()
    for nh in (1, 2, 8):
        for call in (_flash_fwd, _flash_bwd):
            assert call(lib, p, S=0, C=D * nh, nh=nh) == -1
            assert b'empty problem' in lib.og_last_error(), lib.og_last_error()
        for call in (_long_fwd, _long_bwd):
            assert call(lib, p + 1, p, C=D * nh, nh=nh) == -1
            assert b'aligned' in lib.og_last_error(), lib.og_last_error()


def test_other_widths_are_still_refused():
    lib, p = _lib_and_ptr()
    for C in (64, 96, 192, 384):     # d_head 32, 48, 96, 192 at two heads
        for call in (_flash_fwd, _flash_bwd):
            assert call(lib, p, C=C) == -1 and b'd_head = 64' in lib.og_last_error()
    for C in (64, 96, 192):          # d_head 32, 48, 96
        for call in (_long_fwd, _long_bwd):
            assert call(lib, p, p, C=C) == -2 and b'd_head=%d' % (C // 2) in lib.og_last_error()
    # the per-pixel kernels (T <= 32) keep refusing 128
    assert lib.og_temporal_attn_fwd(p, p, p, None, p, 1, 8, 4, 256, 2, 1.0, 0, None) == -2
    assert b'd_head=128' in lib.og_last_error()
    assert lib.og_temporal_attn_bwd(p, p, p, p, p, p, p, None, None, 1, 8, 4, 256, 2, 1.0, 0, None) == -2
    assert b'd_head=128' in lib.og_last_error()


def test_module_accepts_d_head_128_only_besides_64():
    from open_genie_b200.module.attention import SpaceTimeAttention, SpatialAttention, TemporalAttention
    for cls in (SpatialAttention, TemporalAttention):
        m = cls(n_head=2, d_head=128)
        assert m.d_head == 128 and m.scale == 2 * 128 ** -0.5
        for d in (32, 96):
            with pytest.raises(NotImplementedError, match='64 or 128'):
                cls(n_head=2, d_head=d)
    m = SpaceTimeAttention(n_head=(2, 1), d_head=(64, 128))
    assert m.space_attn.n_head == 2 and m.temp_attn.d_head == 128 and m.ffn[1].net[0].num_groups == 1


def test_time_attention_dispatch_rule():
    from open_genie_b200 import ops
    assert not ops._time_attn_tiled(32, 128, 2) and ops._time_attn_tiled(33, 128, 2)
    for T in (1, 16, 32, 33, 200):
        assert ops._time_attn_tiled(T, 256, 2) and ops._time_attn_tiled(T, 128, 1)


# ------------------------------------------------------------------------------------------------------------------
# flash attention, kernel level
# ------------------------------------------------------------------------------------------------------------------
def flash128_run(nseq, S, nh, seed, amp=0.5, aliased=False):
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
@pytest.mark.parametrize('nh', [1, 2])
@pytest.mark.parametrize('S', [1, 16, 63, 65, 100, 257])
def test_flash128_ragged_S(S, nh):
    flash128_run(nseq=3, S=S, nh=nh, seed=30000 + 10 * S + nh)


@GPU
def test_flash128_full_size_frame():
    flash128_run(nseq=1, S=4096, nh=2, seed=30500)


@GPU
def test_flash128_eight_heads():
    """C = 1024: head h reads and writes columns [128 h, 128 h + 128)."""
    flash128_run(nseq=2, S=130, nh=8, seed=30600)


@GPU
@pytest.mark.parametrize('S,nh', [(100, 2), (256, 4)])
def test_flash128_aliased_product_call(S, nh):
    flash128_run(nseq=2, S=S, nh=nh, seed=30700 + S, aliased=True)


# ------------------------------------------------------------------------------------------------------------------
# tiled temporal attention, kernel level
# ------------------------------------------------------------------------------------------------------------------
def long128_run(B, T, P, nh, bcast, seed, amp=1.0, aliased=False, do_mask=None, check_guards=True):
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
@pytest.mark.parametrize('T', [1, 2, 15, 16, 17, 32, 33, 64, 65, 200])
def test_long128_kernels(T, bcast):
    long128_run(2, T, 5, 2, bcast, seed=31000 + 10 * T + bcast)


@GPU
def test_long128_aliased_product_call():
    long128_run(2, 100, 6, 2, 0, seed=31500, aliased=True)


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_long128_large_scores(bcast):
    """|scale q.k| far beyond 89 in places: the online rescale must keep exp in range from tile to tile."""
    B, T, P, nh = 2, 130, 4, 2
    inp, _ = long128_run(B, T, P, nh, bcast, seed=31600 + bcast, amp=3.5)
    qs = _tseq(inp['q'].float(), nh)
    ks = _kvseq(inp['k'].float(), nh) if bcast else _tseq(inp['k'].float(), nh)
    s = ((nh * D ** -0.5) * (qs @ ks.transpose(-1, -2))).tril()
    assert s.abs().amax().item() > 89, 'scores too small to overflow exp without the max subtraction'


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_long128_T1_is_exact(bcast):
    """One time step: the softmax is exactly 1, so out = v (+ residual, rounded once) and, without broadcast, dv = dout."""
    B, T, P, nh = 2, 1, 9, 2
    inp, got = long128_run(B, T, P, nh, bcast, seed=31700 + bcast)
    v = inp['v']
    vb = v[:, :, None].expand(B, T, P, nh * D) if bcast else v
    assert torch.equal(got['out'], vb)
    assert torch.equal(got['out_res'], (vb.float() + inp['res'].float()).to(BF16))
    if not bcast:
        assert torch.equal(got['dv'], inp['do'])


@GPU
@pytest.mark.parametrize('T,bcast', [(150, 0), (150, 1), (20, 0)])
def test_long128_causality_is_exact(T, bcast):
    """Changing every input row t' > t0 (q, k and v) leaves output rows <= t0 bit-identical: out, out_res and lse."""
    B, P, nh = 2, 6, 2
    C, scale = nh * D, nh * D ** -0.5
    kvshape = (B, T, C) if bcast else (B, T, P, C)
    q, k, v, res = _rand((B, T, P, C), 32000), _rand(kvshape, 32001), _rand(kvshape, 32002), _rand((B, T, P, C), 32003)
    t0 = T // 2 + 3
    q2, k2, v2 = q.clone(), k.clone(), v.clone()
    for t, s in ((q2, 32004), (k2, 32005), (v2, 32006)):
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
def test_long128_bcast_gradient_many_pixel_chunks():
    """kv_bcast = 1 at P = 4096: every (b, h) is split into many pixel chunks, each added into dK / dV on its own; a
    second pass has dO non-zero only on the first two and last two pixels, so a lost or misrouted chunk is caught."""
    B, T, P, nh = 2, 40, 4096, 2
    long128_run(B, T, P, nh, 1, seed=32100)
    edge = torch.zeros(P, device=DEV, dtype=BF16)
    edge[[0, 1, P - 2, P - 1]] = 1
    long128_run(B, T, P, nh, 1, seed=32200, do_mask=edge.view(1, 1, P, 1), check_guards=False)


# ------------------------------------------------------------------------------------------------------------------
# which kernels run at d_head = 128
# ------------------------------------------------------------------------------------------------------------------
FLASH128 = ['og_flash_attn_fwd_d128_kernel', 'og_flash_attn_bwd_d128_kernel<0>', 'og_flash_attn_bwd_d128_kernel<1>',
            'og_attn_delta_d128_kernel']
LONG128 = ['og_temporal_attn_long_fwd_kernel<128>', 'og_temporal_attn_long_bwd_dq_kernel<128>',
           'og_temporal_attn_long_bwd_dkdv_kernel<128>']


@GPU
def test_flash128_kernel_names():
    names = [n for n in _kernels_run(lambda: flash128_run(nseq=1, S=65, nh=1, seed=33000)) if 'og_' in n]
    for w in FLASH128:
        assert any(w in n for n in names), (w, sorted(set(names)))
    for a in ('og_flash_attn_fwd_kernel', 'og_flash_attn_bwd_kernel<', 'og_attn_delta_kernel'):
        assert not any(a in n for n in names), (a, sorted(set(names)))


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_time_attention_d128_runs_the_tiled_kernels(T):
    from open_genie_b200 import ops
    B, H, W, nh = 1, 4, 4, 2
    C = D * nh
    x = _rand((B, T, H, W, C), 33100 + T).requires_grad_(True)
    freq = O.rope_freq(C, '1d').to(DEV)
    gamma = torch.ones(C, device=DEV, requires_grad=True)
    beta = torch.zeros(C, device=DEV, requires_grad=True)

    def run():
        y = ops.time_attention_res(x, freq, gamma, beta, nh, nh * D ** -0.5)
        y.backward(torch.ones_like(y))
    names = [n for n in _kernels_run(run) if 'og_' in n]
    for w in LONG128:
        assert any(w in n for n in names), (T, w, sorted(set(names)))
    for a in ('og_temporal_attn_fwd_kernel<', 'og_temporal_attn_bwd_kernel<', '_mma_kernel', '_kernel<64>'):
        assert not any(a in n for n in names), (T, a, sorted(set(names)))


# ------------------------------------------------------------------------------------------------------------------
# model level, against the CPU oracle
# ------------------------------------------------------------------------------------------------------------------
def _grads(m):
    return {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}


def _ref_sd(sd):
    return {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith(('freq', 'bit_mask')))
            for k, v in sd.items()}


def _check_block(m, ref_fn, sd, shape, tag, cond_dim):
    x = O.det_uniform(tag + '.x', shape)
    gy = O.det_uniform(tag + '.gy', shape, 1e-3)
    cond = O.det_uniform(tag + '.cond', (shape[0], shape[1], cond_dim)).sign() if cond_dim else None
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
@pytest.mark.parametrize('nh', [1, 2])
def test_spacetime_block_d128_against_oracle(nh, cond_dim, T):
    from open_genie_b200.module.attention import SpaceTimeAttention
    kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
    m = SpaceTimeAttention(n_head=nh, d_head=D, transpose=False, **kw)
    sd = det_weights(m)
    m.to(DEV)
    _check_block(m, lambda s, x, c: O.spacetime_attention(s, '', x, nh, False, c), sd, (2, T, 4, 4, D * nh),
                 f'd128.st.{nh}.{cond_dim}.{T}', cond_dim)


@GPU
@pytest.mark.parametrize('T', [16, 40])
def test_mixed_width_block_against_oracle(T):
    """Space attention with 2 heads of 64, time attention with 1 head of 128, on the same 128 channels (the FFN's
    GroupNorm takes the temporal head count)."""
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=(2, 1), d_head=(64, D), transpose=False)
    sd = det_weights(m)
    m.to(DEV)

    def ref(s, x, cond):
        x = O.spatial_attention(s, 'space_attn.', x, 2, False) + x
        x = O.temporal_attention(s, 'temp_attn.', x, 1, False, cond) + x
        y = F.group_norm(x.movedim(-1, 1), 1, s['ffn.1.net.0.weight'], s['ffn.1.net.0.bias'], 1e-5)
        return F.conv3d(y, s['ffn.1.net.1.0.weight'], None, padding=1).movedim(1, -1) + x
    _check_block(m, ref, sd, (2, T, 4, 4, D), f'd128.mixed.{T}', None)


def _dyn_inputs(T, hw, vocab, act_vocab, tag):
    shape = (2, T, hw, hw)
    u = O.det_uniform(f'{tag}.tokens', shape) / (3 ** 0.5)
    tokens = ((u + 1) * 0.5 * vocab).long().clamp(0, vocab - 1)
    ua = O.det_uniform(f'{tag}.act', shape[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * act_vocab).long().clamp(0, act_vocab - 1)
    mask = O.det_uniform(f'{tag}.mask', shape) / (3 ** 0.5) < 0.5
    return tokens, act, mask


@GPU
@pytest.mark.parametrize('T,embed,nh,hw', [(4, 128, 1, 8), (40, 128, 1, 8), (16, 512, 4, 16)])
def test_dynamics_d128_against_oracle(T, embed, nh, hw):
    import open_genie_b200 as og
    desc = (('space-time_attn', {'n_rep': 2, 'n_head': nh, 'd_head': D, 'transpose': False}),)
    kw = dict(fx.MINI_DYN, embed_dim=embed)
    dm = og.DynamicsModel(desc, **kw)
    sd = det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = _dyn_inputs(T, hw, kw['tok_vocab'], kw['act_vocab'], f'd128.dyn.{T}.{embed}')
    ref_sd = _ref_sd(sd)
    ref_loss = O.dynamics_loss(ref_sd, desc, tokens, act, mask)
    ref_loss.backward()
    loss = dm.compute_loss(tokens.to(DEV), act.to(DEV), mask=mask.to(DEV))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) / ref_loss.item() < 2e-2
    for k, g in _grads(dm).items():
        r = ref_sd[k].grad
        assert r is not None, k
        assert rel_l2(g, r) < 0.1, (k, rel_l2(g, r))


@GPU
def test_latent_action_d128_against_oracle():
    """Every space-time block with one head of 128; the decoder's temporal attention takes K / V from the action codes
    (the broadcast-K/V path of the tiled kernels, which d_head = 128 runs at every T)."""
    import open_genie_b200 as og
    wide = lambda bp: tuple((n, {**kw, 'n_head': 1, 'd_head': D} if n == 'space-time_attn' else kw) for n, kw in bp)
    enc, dec = wide(fx.MINI_ACT_ENC), wide(fx.MINI_ACT_DEC)
    la = og.LatentAction(enc, dec, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    la.to(DEV).train()
    video = O.det_uniform('d128.action.video', fx.MINI_ACT_VIDEO_SHAPE)
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
def test_spacetime_block_d128_cuda_graph_replay_matches_eager():
    from open_genie_b200.module.attention import SpaceTimeAttention
    m = SpaceTimeAttention(n_head=2, d_head=D, transpose=False)
    det_weights(m)
    m.to(DEV)
    shape = (2, 16, 4, 4, 2 * D)
    x = O.det_uniform('d128.graph.x', shape).to(DEV).requires_grad_(True)
    gy = O.det_uniform('d128.graph.gy', shape, 1e-3).to(DEV)

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
