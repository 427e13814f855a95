"""Temporal attention beyond 32 frames: og_temporal_attn_long_fwd / bwd (csrc/temporal_attn_long.cu), the T > 32 path of
ops._TimeAttnFn, and the models that run it.

Kernel level: every output element against the float64 reference of test_gpu_attention_paths, with the rounding model
of an online-softmax kernel (P and dS in bf16, delta from the stored bf16 output), at tile edges from T = 1 to 1024.
Model level: SpaceTimeAttention, DynamicsModel, LatentAction and Genie at T > 32 against the CPU oracle (which runs
SDPA and takes any T), with the tolerances of the T = 16 golden tests.
"""
import ctypes

import pytest
import torch

from helpers import det_weights, rel_l2
from oracle import fixtures as fx
from oracle import genie_oracle as O
from test_gpu_attention_paths import (BF16, DEV, F32T, SLACK, U, Guarded, _call, _kernels_run, _kvseq, _kvsum, _rand,
                                      _tseq, _tunseq, attn_err, attn_ref, bf16_tol, check_all, gam)

GPU = pytest.mark.gpu
LONG_KERNELS = ['og_temporal_attn_long_fwd_kernel', 'og_temporal_attn_long_bwd_dkdv_kernel',
                'og_temporal_attn_long_bwd_dq_kernel']


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation (no device needed)
# ------------------------------------------------------------------------------------------------------------------
def _lib_and_ptr():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    return lib, ctypes.addressof(buf)


def _fwd(lib, p, B=1, T=40, P=4, C=128, nh=2, scale=1.0, q='p', res=None, out_res=None, lse='p'):
    a = {'p': p, None: None}
    return lib.og_temporal_attn_long_fwd(a[q], p, p, p, res, out_res, a[lse], B, T, P, C, nh, scale, 0, None)


def _bwd(lib, p, B=1, T=40, P=4, C=128, nh=2, scale=1.0, bcast=0, lse='p', dk='p'):
    a = {'p': p, None: None}
    return lib.og_temporal_attn_long_bwd(p, p, p, p, p, a[lse], p, p, a[dk], a[dk], None, None, B, T, P, C, nh, scale,
                                         bcast, None)


def test_long_argument_validation_returns_status_codes():
    lib, p = _lib_and_ptr()
    # null pointers
    assert _fwd(lib, p, q=None) == -1 and b'null pointer' in lib.og_last_error()
    assert _fwd(lib, p, lse=None) == -1
    assert _bwd(lib, p, lse=None) == -1 and b'null pointer' in lib.og_last_error()
    assert _bwd(lib, p, dk=None) == -1 and b'missing dk/dv' in lib.og_last_error()
    assert _bwd(lib, p, bcast=1) == -1 and b'missing dk/dv' in lib.og_last_error()    # no dk_bcast / dv_bcast
    # a residual without out_res, and the reverse
    assert _fwd(lib, p, res=p) == -1 and b'together' in lib.og_last_error()
    assert _fwd(lib, p, out_res=p) == -1
    # empty problems
    for B, T, P in ((1, 0, 4), (0, 40, 4), (1, 40, 0), (-1, 40, 4)):
        assert _fwd(lib, p, B=B, T=T, P=P) == -1 and b'empty problem' in lib.og_last_error()
        assert _bwd(lib, p, B=B, T=T, P=P) == -1 and b'empty problem' in lib.og_last_error()
    # C not a multiple of n_head
    assert _fwd(lib, p, C=129) == -1 and _bwd(lib, p, C=129) == -1
    # d_head 48 (and 32): unsupported shape
    for C in (96, 64):
        assert _fwd(lib, p, C=C) == -2 and b'd_head=%d' % (C // 2) in lib.og_last_error()
        assert _bwd(lib, p, C=C) == -2 and b'd_head=%d' % (C // 2) in lib.og_last_error()
    # non-positive scale
    for scale in (0.0, -1.0):
        assert _fwd(lib, p, scale=scale) == -1 and b'scale' in lib.og_last_error()
        assert _bwd(lib, p, scale=scale) == -1 and b'scale' in lib.og_last_error()


# ------------------------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------------------------
def long_expect(q, k, v, do, res, nh, scale, bcast, dk_init=None, dv_init=None):
    """{output: (reference, tolerance)} of og_temporal_attn_long_fwd / bwd on these bf16 inputs, in the kernels'
    layouts. q, do, res: [B, T, P, C]; k, v: the same (bcast = 0) or [B, T, C] (bcast = 1)."""
    B, T, P, C = q.shape
    f = lambda t: t.double()
    qs, dos = _tseq(f(q), nh), _tseq(f(do), nh)
    ks, vs = (_kvseq(f(k), nh), _kvseq(f(v), nh)) if bcast else (_tseq(f(k), nh), _tseq(f(v), nh))
    r = attn_ref(qs, ks, vs, scale, causal=True, do=dos)
    e = attn_err(qs, ks, vs, r, scale, p_bf16=True, do=dos, delta_from_bf16_o=True)
    o, eo = _tunseq(r['o']), _tunseq(e['o'])
    out = {'out': (o, bf16_tol(eo, o))}
    orr = o + f(res)
    out['out_res'] = (orr, SLACK * (eo + U * orr.abs()))            # added in fp32, rounded once
    out['lse'] = (r['lse'].permute(0, 2, 1, 3), SLACK * e['lse'].permute(0, 2, 1, 3))   # [B, nh, P, T]
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


def long_run(B, T, P, nh, bcast, seed, amp=1.0, aliased=False, do_mask=None, check_guards=True):
    """og_temporal_attn_long_fwd (with a residual) and og_temporal_attn_long_bwd on guarded outputs, every output
    checked against `long_expect`. The broadcast K/V gradients start from non-zero values."""
    C, scale = nh * 64, nh * 64 ** -0.5
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
    return {'q': q, 'k': k, 'v': v}, {n: o.t for n, o in outs.items()}


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('T', [1, 16, 17, 33, 47, 64, 65, 128, 200, 1024])
def test_long_kernels(T, bcast):
    """Tile edges: one partial tile (1, 16, 17, 33, 47), exactly one (64), one row into the second (65), two full
    tiles (128), a ragged fourth (200) and sixteen tiles (1024)."""
    B, P, nh = (1, 3, 2) if T > 256 else (2, 5, 2)
    long_run(B, T, P, nh, bcast, seed=20000 + 10 * T + bcast)


@GPU
def test_long_aliased_product_call():
    """q = k = v, as _TimeAttnFn makes the call: dq, dk and dv are the three partial gradients of one tensor."""
    long_run(2, 100, 6, 2, 0, seed=21000, aliased=True)


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_long_large_scores(bcast):
    """|scale q.k| far beyond 89 in places: the online rescale must keep exp in range from tile to tile."""
    B, T, P, nh = 2, 130, 4, 2
    inp, _ = long_run(B, T, P, nh, bcast, seed=22000 + bcast, amp=4.5)
    qs = _tseq(inp['q'].float(), nh)
    ks = _kvseq(inp['k'].float(), nh) if bcast else _tseq(inp['k'].float(), nh)
    s = ((nh * 64 ** -0.5) * (qs @ ks.transpose(-1, -2))).tril()
    assert s.abs().amax().item() > 89, 'scores too small to overflow exp without the max subtraction'


@GPU
def test_long_bcast_gradient_many_pixel_chunks():
    """kv_bcast = 1 at P = 4096: every (b, h) is split into many pixel chunks (the last one ragged), each added into
    dK / dV on its own. A second backward pass has dO non-zero only on the first two and last two pixels of every
    (b, h), so a lost or misrouted chunk is far outside the bound."""
    B, T, P, nh = 2, 40, 4096, 4
    long_run(B, T, P, nh, 1, seed=23000)
    edge = torch.zeros(P, device=DEV, dtype=BF16)
    edge[[0, 1, P - 2, P - 1]] = 1
    long_run(B, T, P, nh, 1, seed=23100, do_mask=edge.view(1, 1, P, 1), check_guards=False)


@GPU
@pytest.mark.parametrize('T,bcast', [(150, 0), (150, 1), (70, 0)])
def test_long_causality_is_exact(T, bcast):
    """Changing every input row t' > t0 (q, k and v) leaves output rows <= t0 bit-identical: out, out_res and lse."""
    B, P, nh = 2, 6, 2
    C, scale = nh * 64, nh * 64 ** -0.5
    kvshape = (B, T, C) if bcast else (B, T, P, C)
    q, k, v, res = _rand((B, T, P, C), 24000), _rand(kvshape, 24001), _rand(kvshape, 24002), _rand((B, T, P, C), 24003)
    t0 = T // 2 + 3
    q2, k2, v2 = q.clone(), k.clone(), v.clone()
    for t, s in ((q2, 24004), (k2, 24005), (v2, 24006)):
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
@pytest.mark.parametrize('T', [32, 33])
def test_time_attention_dispatch_by_clip_length(T):
    """ops.time_attention_res keeps today's kernels up to T = 32 and runs the three tiled kernels from T = 33 on."""
    from open_genie_b200 import ops
    B, H, W, nh = 1, 4, 4, 2
    C = 64 * nh
    x = _rand((B, T, H, W, C), 25000).requires_grad_(True)
    freq = O.rope_freq(C, '1d').to(DEV)
    gamma = torch.ones(C, device=DEV, requires_grad=True)
    beta = torch.zeros(C, device=DEV, requires_grad=True)

    def run():
        y = ops.time_attention_res(x, freq, gamma, beta, nh, nh * 64 ** -0.5)
        y.backward(torch.ones_like(y))
    names = [n for n in _kernels_run(run) if 'og_' in n]
    old = ['og_temporal_attn_fwd_kernel<64>', 'og_temporal_attn_bwd_kernel<64>']
    want, absent = (old, ['_long_']) if T <= 32 else (LONG_KERNELS, ['og_temporal_attn_fwd_kernel<',
                                                                      'og_temporal_attn_bwd_kernel<', '_mma_kernel'])
    for w in want:
        assert any(w in n for n in names), (T, w, sorted(set(names)))
    for a in absent:
        assert not any(a in n for n in names), (T, a, sorted(set(names)))


# ------------------------------------------------------------------------------------------------------------------
# model level, against the CPU oracle (tolerances of the T = 16 golden tests)
# ------------------------------------------------------------------------------------------------------------------
def _grads(m):
    return {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}


def _st_block(cond_dim):
    from open_genie_b200.module.attention import SpaceTimeAttention
    kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
    m = SpaceTimeAttention(n_head=2, d_head=64, transpose=False, **kw)
    sd = det_weights(m)
    return m.to(DEV), sd


@GPU
@pytest.mark.parametrize('cond_dim', [None, 4])
def test_spacetime_block_T48_against_oracle(cond_dim):
    m, sd = _st_block(cond_dim)
    shape = (2, 48, 4, 4, 128)
    tag = f'long.st.{cond_dim}'
    x = O.det_uniform(tag + '.x', shape)
    gy = O.det_uniform(tag + '.gy', shape, 1e-3)
    cond = O.det_uniform(tag + '.cond', (2, 48, 4)).sign() if cond_dim else None
    xr = x.clone().requires_grad_(True)
    ref_sd = {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith('freq')) for k, v in sd.items()}
    yr = O.spacetime_attention(ref_sd, '', xr, 2, False, cond)
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


def _dyn_inputs(T):
    shape = (2, T, 8, 8)
    u = O.det_uniform(f'long.dyn.tokens.{T}', shape) / (3 ** 0.5)
    tokens = ((u + 1) * 0.5 * fx.MINI_DYN['tok_vocab']).long().clamp(0, fx.MINI_DYN['tok_vocab'] - 1)
    ua = O.det_uniform(f'long.dyn.act.{T}', shape[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * fx.MINI_DYN['act_vocab']).long().clamp(0, fx.MINI_DYN['act_vocab'] - 1)
    mask = O.det_uniform(f'long.dyn.mask.{T}', shape) / (3 ** 0.5) < 0.5
    return tokens, act, mask


@GPU
def test_dynamics_compute_loss_T40_against_oracle():
    import open_genie_b200 as og
    dm = og.DynamicsModel(fx.MINI_DYN_DESC, **fx.MINI_DYN)
    sd = det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = _dyn_inputs(40)
    ref_sd = {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith('freq')) for k, v in sd.items()}
    ref_loss = O.dynamics_loss(ref_sd, fx.MINI_DYN_DESC, tokens, act, mask)
    ref_loss.backward()
    loss = dm.compute_loss(tokens.to(DEV), act.to(DEV), mask=mask.to(DEV))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) / ref_loss.item() < 2e-2
    for k, g in _grads(dm).items():
        r = ref_sd[k].grad
        assert r is not None, k
        assert rel_l2(g, r) < 0.1, (k, rel_l2(g, r))


@GPU
def test_latent_action_T36_against_oracle():
    """The decoder's temporal attention takes its K / V from the action codes: the broadcast-K/V path at T = 36."""
    import open_genie_b200 as og
    la = og.LatentAction(fx.MINI_ACT_ENC, fx.MINI_ACT_DEC, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    la.to(DEV).train()
    shape = fx.MINI_ACT_VIDEO_SHAPE[:2] + (36,) + fx.MINI_ACT_VIDEO_SHAPE[3:]
    video = O.det_uniform('long.action.video', shape)
    ref_sd = {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith(('freq', 'bit_mask')))
              for k, v in sd.items()}
    _, ref_loss, (ref_rec, _), _ = O.latent_action_forward(ref_sd, fx.MINI_ACT_ENC, fx.MINI_ACT_DEC, video,
                                                           fx.MINI_ACT_D_CODEBOOK)
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
def test_genie_rolls_out_34_frames_from_one_image():
    """Genie.forward runs the dynamics model on t + 1 frames for every generated frame: up to T = 35 here."""
    import open_genie_b200 as og
    torch.manual_seed(0)
    no_time = lambda bp: tuple((n, {**kw, **({'time_factor': 1} if 'time_factor' in kw else {})}) for n, kw in bp)
    tok = og.VideoTokenizer(no_time(fx.MINI_ENC), no_time(fx.MINI_DEC), d_codebook=fx.MINI_D_CODEBOOK, gan_loss_weight=0,
                            perc_loss_weight=0)
    gen = og.Genie(tok,
                   dict(enc_desc=fx.MINI_ACT_ENC, dec_desc=fx.MINI_ACT_DEC, d_codebook=4, n_embd=128, inp_shape=(32, 32)),
                   dict(desc=fx.MINI_DYN_DESC, tok_vocab=2 ** fx.MINI_D_CODEBOOK, act_vocab=16, embed_dim=128)).to(DEV)
    prompt = torch.randn(2, 3, 32, 32, device=DEV)
    actions = torch.randint(0, 16, (2, 34), device=DEV)
    video = gen(prompt, actions, num_frames=34, steps_per_frame=2)
    assert video.shape == (2, 3, 35, 32, 32) and video.dtype == torch.float32 and torch.isfinite(video).all()


@GPU
def test_dynamics_generate_40_frames_is_self_consistent():
    """generate on a 40-frame history (the transformer runs at T = 41) returns the sampler's tokens for the model's own
    last-frame logits."""
    import open_genie_b200 as og
    from open_genie_b200 import ops
    dm = og.DynamicsModel(fx.MINI_DYN_DESC, **fx.MINI_DYN)
    det_weights(dm)
    dm.to(DEV)
    tokens, act, _ = _dyn_inputs(40)
    tokens, act = tokens.to(DEV), act.to(DEV)
    steps = 5
    uni = torch.rand((steps, 2 * 64), generator=torch.Generator(device=DEV).manual_seed(26000), device=DEV)
    out = dm.generate(tokens, act, steps=steps, uniforms=uni)
    assert out.shape == (2, 41, 8, 8) and torch.equal(out[:, :40], tokens)
    tok_id = torch.cat([tokens, torch.zeros(2, 1, 8, 8, dtype=tokens.dtype, device=DEV)], 1)
    act_id = torch.cat([act, torch.zeros(2, 1, dtype=act.dtype, device=DEV)], 1)
    code, _ = ops.maskgit_sample(dm._logits(tok_id, act_id)[:, -1], uni, dm.get_schedule(steps, (8, 8)))
    assert torch.equal(out[:, -1], code)


@GPU
def test_spacetime_block_T48_cuda_graph_replay_matches_eager():
    """Forward + backward of one block at T = 48 captured in a CUDA graph after a warm-up: the tiled temporal kernels
    make no host synchronisation and allocate only through torch."""
    m, _ = _st_block(None)
    shape = (2, 48, 4, 4, 128)
    x = O.det_uniform('long.graph.x', shape).to(DEV).requires_grad_(True)
    gy = O.det_uniform('long.graph.gy', shape, 1e-3).to(DEV)

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
