"""SpaceTimeAttention feed-forward blocks beyond GroupNorm -> one conv: hidden layers with GELU (`hid_dim`), a width
change with the 1x1x1 `ffn_skip` conv (`d_out`, transpose=True), conv biases (`bias=True`) and kernel size 1.

CPU: state_dict keys and shapes against the reference's (tests/golden/st_block_ffn.pt, written by
oracle/make_golden_ffn.py), the restatement oracle/ffn_oracle.py against the reference's outputs, the refusals, and the
argument checks of og_gelu_fwd / og_gelu_bwd.
GPU: the GELU kernels element by element against float64; the convolution entry points at the new widths (512 -> 2048
-> 512 channels at k = 3) exactly on small-integer operands; blocks, DynamicsModel and LatentAction against the oracle;
CUDA-graph replay and the zero arena.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import Guarded, det_weights, rel_l2
from oracle import ffn_oracle as FO
from oracle import fixtures as fx
from oracle import genie_oracle as O

GPU = pytest.mark.gpu
DEV = 'cuda'
BF16 = torch.bfloat16
GOLDEN = 'st_block_ffn.pt'
CASES = ('hid512', 'hid256_384_t1', 'dout256_t1', 'dout256_hid512_t1', 'bias', 'bias_cond', 'bias_hid256_cond_t1',
         'hid512_k1')


def _block(**kw):
    from open_genie_b200.module.attention import SpaceTimeAttention
    return SpaceTimeAttention(**kw)


def _golden_inputs(tag, c):
    shape = c['shape']
    x = O.det_uniform(f'stffn.x.{tag}', shape)
    cond_dim = c['kw'].get('time_attn_kw', {}).get('key_dim')
    t = shape[2] if c['kw'].get('transpose', False) else shape[1]
    cond = O.det_uniform(f'stffn.cond.{tag}', (shape[0], t, cond_dim)).sign() if cond_dim else None
    return x, cond


def _sample(key, t, n):
    """The elements oracle/make_golden_ffn.py stored of `t`."""
    return t.detach().float().cpu().flatten()[O.det_indices(key, t.numel(), n)]


def _golden_grads(tag, c, grads):
    """(name, sample of the gradient, stored sample, stored norm) for every gradient of a golden case."""
    n = c['grad'].numel() // len(c['grad_names'])
    return [(k, _sample(f'stffn.g.{tag}.{k}', grads[k], n), c['grad'][i * n:(i + 1) * n], c['grad_norm'][k])
            for i, k in enumerate(c['grad_names'])]


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def test_golden_holds_every_case(golden):
    assert tuple(golden(GOLDEN)) == CASES


@pytest.mark.parametrize('tag', CASES)
def test_state_dict_matches_reference(golden, tag):
    c = golden(GOLDEN)[tag]
    m = _block(n_head=2, d_head=64, **c['kw'])
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == c['keys']
    assert m.out_channels == c['y_shape'][1 if c['kw'].get('transpose', False) else -1]


@pytest.mark.parametrize('tag', CASES)
def test_oracle_reproduces_reference(golden, tag):
    c = golden(GOLDEN)[tag]
    sd = det_weights(_block(n_head=2, d_head=64, **c['kw']))
    ref = {k: v.clone().requires_grad_(not k.endswith('freq')) for k, v in sd.items()}
    x, cond = _golden_inputs(tag, c)
    x.requires_grad_(True)
    y = FO.spacetime_attention(ref, '', x, 2, c['kw'].get('transpose', False), cond)
    y.square().mean().backward()
    assert tuple(y.shape) == c['y_shape']
    n = c['y'].numel()
    torch.testing.assert_close(_sample(f'stffn.y.{tag}', y, n), c['y'], rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(_sample(f'stffn.dx.{tag}', x.grad, n), c['dx'], rtol=2e-4, atol=1e-6)
    grads = {k: v.grad for k, v in ref.items() if v.grad is not None}
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads(tag, c, grads):
        torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-6)
        assert abs(grads[k].norm().item() - norm) <= 1e-4 * norm + 1e-7, k


def test_oracle_default_block_is_the_existing_restatement():
    """Without hidden layers, biases or ffn_skip, ffn_oracle computes what oracle.genie_oracle computes."""
    for transpose, cond_dim, shape in fx.ST_BLOCK_CASES[2:]:
        kw = {'time_attn_kw': {'key_dim': cond_dim}} if cond_dim else {}
        sd = det_weights(_block(n_head=2, d_head=64, transpose=transpose, **kw))
        x = O.det_uniform('ffn.default.x', shape)
        cond = O.det_uniform('ffn.default.cond', (shape[0], shape[1], cond_dim)).sign() if cond_dim else None
        assert torch.equal(FO.spacetime_attention(sd, '', x, 2, transpose, cond),
                           O.spacetime_attention(sd, '', x, 2, transpose, cond))


def test_refusals():
    with pytest.raises(NotImplementedError, match='d_inp'):
        _block(n_head=2, d_head=64, d_inp=64)
    with pytest.raises(NotImplementedError, match='transpose=True'):
        _block(n_head=2, d_head=64, d_out=256)
    for kw in ({'hid_dim': 100}, {'hid_dim': (512, 96)}, {'hid_dim': 0}, {'d_out': 160, 'transpose': True}):
        with pytest.raises(NotImplementedError, match='multiples of 64'):
            _block(n_head=2, d_head=64, **kw)
    # what the reference accepts as no-ops
    m = _block(n_head=2, d_head=64, d_inp=128, d_out=128, hid_dim=[256])
    assert m.in_channels == m.out_channels == 128 and len(m.ffn[1].net) == 3


def test_gelu_entry_points_validate_arguments():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    p = (ctypes.addressof(buf) + 15) & ~15

    def fwd(u=p, a=p, rows=4, C=8):
        return lib.og_gelu_fwd(u, a, rows, C, None)

    def bwd(da=p, u=p, du=p, rows=4, C=8):
        return lib.og_gelu_bwd(da, u, du, rows, C, None)
    for call, ptrs in ((fwd, ('u', 'a')), (bwd, ('da', 'u', 'du'))):
        for name in ptrs:
            assert call(**{name: None}) == -1 and b'null pointer' in lib.og_last_error()
            assert call(**{name: p + 8}) == -1 and b'16-byte aligned' in lib.og_last_error()
        for C in (0, 4, 12, -8):
            assert call(C=C) == -1 and b'multiple of 8' in lib.og_last_error()
        for rows in (0, -1):
            assert call(rows=rows) == -1 and b'empty problem' in lib.og_last_error()


# ------------------------------------------------------------------------------------------------------------------
# GELU kernels against float64
# ------------------------------------------------------------------------------------------------------------------
def _ulp_bf16(r):
    """One bf16 ulp at |r| (float64): 2^(e - 7) for 2^e <= |r| < 2^(e+1), and 2^-133 below the normal range and at 0."""
    _, e = torch.frexp(r.abs())
    return torch.ldexp(torch.ones_like(r), torch.where(r == 0, -133, (e - 8).clamp_min(-133)))


def _gelu64(u):
    cdf = 0.5 * torch.special.erfc(-u / math.sqrt(2.0))
    pdf = torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)
    return u * cdf, cdf + u * pdf, cdf + u.abs() * pdf


SPECIAL = [0.0, -0.0, 1e-30, -1e-30, 1e-39, -1e-39, 1e-3, -1e-3, 0.5, -0.5, -0.7518, 1.0, -1.0, 3.0, -3.0, 5.5, -5.5,
           9.9, -9.9, 10.0, -10.0, -13.0, -15.0, -20.0, -40.0, -1e4]


@GPU
@pytest.mark.parametrize('C', [8, 24, 520, 2048])
@pytest.mark.parametrize('rows', [1, 7, 333])
def test_gelu_kernels_against_float64(rows, C):
    """Forward: every element within one bf16 ulp of float64 GELU of the same bf16 input, and -0 where u << 0.
    Backward: |du - da GELU'(u)| <= ulp_bf16(ref) + 2^-20 |da| (Phi(u) + |u| phi(u)): the output rounding, plus fp32
    evaluation of erfc / exp / the products (a few fp32 ulps of the terms) where the two terms cancel (u ~ -0.75)."""
    g = torch.Generator().manual_seed(7000 + rows * 4096 + C)
    u = (torch.randn(rows, C, generator=g, dtype=torch.float64) * 3.5).clamp(-10.5, 10.5)
    flat = u.view(-1)
    k = min(len(SPECIAL), flat.numel())
    flat[:k] = torch.tensor(SPECIAL[:k], dtype=torch.float64)
    da = torch.randn(rows, C, generator=g, dtype=torch.float64) * 2.0
    ub, dab = u.to(BF16).to(DEV), da.to(BF16).to(DEV)
    a, du = Guarded((rows, C), BF16), Guarded((rows, C), BF16)
    s = torch.cuda.current_stream().cuda_stream
    from open_genie_b200 import _lib
    _lib.call('og_gelu_fwd', ub.data_ptr(), a.ptr(), rows, C, s)
    _lib.call('og_gelu_bwd', dab.data_ptr(), ub.data_ptr(), du.ptr(), rows, C, s)
    torch.cuda.synchronize()
    a.check_guard('a')
    du.check_guard('du')
    u64, da64 = ub.double().cpu(), dab.double().cpu()
    ref, dref, mag = _gelu64(u64)
    got = a.t.double().cpu()
    err = (got - ref).abs()
    bad = ~(err <= _ulp_bf16(ref))
    assert not bad.any(), (int(bad.sum()), u64[bad][:5].tolist(), got[bad][:5].tolist(), ref[bad][:5].tolist())
    neg = u64 < -15
    assert torch.signbit(a.t.cpu()[neg]).all() and (got[neg] == 0).all()
    gd, rd = du.t.double().cpu(), da64 * dref
    bound = _ulp_bf16(rd) + 2.0 ** -20 * da64.abs() * mag
    bad = ~((gd - rd).abs() <= bound)
    assert not bad.any(), (int(bad.sum()), u64[bad][:5].tolist(), gd[bad][:5].tolist(), rd[bad][:5].tolist())


# ------------------------------------------------------------------------------------------------------------------
# convolution entry points at the FFN's widths: 512 -> 2048 -> 512 channels, k = 3 (K up to 27 * 2048)
# ------------------------------------------------------------------------------------------------------------------
def _ints(shape, seed, lo=-1, hi=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).double()


@GPU
@pytest.mark.parametrize('cin,cout', [(512, 2048), (2048, 512)])
def test_conv_entry_points_at_hidden_widths_are_exact(cin, cout):
    """Operands in {-1, 0, 1}, biases in [-3, 3]: every sum of |terms| is below 27 * 2048 * 2 < 2^22, so the fp32
    accumulation is exact; bf16 outputs must equal the bf16 rounding of the float64 result, fp32 ones must equal it."""
    from open_genie_b200 import _lib
    N, T, H, W, k = 2, 4, 8, 8, 3
    s = torch.cuda.current_stream().cuda_stream
    x = _ints((N, cin, T, H, W), 1 + cin)
    w = _ints((cout, cin, k, k, k), 2 + cin)
    b = _ints((cout,), 3 + cin, -3, 3)
    dy = _ints((N, cout, T, H, W), 4 + cin)
    xd, wd, dyd = x.to(DEV), w.to(DEV), dy.to(DEV)
    y_ref = F.conv3d(xd, wd, b.to(DEV), padding=1)
    dx_ref = torch.nn.grad.conv3d_input(x.shape, wd, dyd, padding=1)
    dw_ref = torch.nn.grad.conv3d_weight(xd, w.shape, dyd, padding=1)
    rows = lambda t: t.permute(0, 2, 3, 4, 1).contiguous()                # NCDHW -> NDHWC
    xr, dyr = rows(xd).to(BF16), rows(dyd).to(BF16)
    packed = wd.permute(0, 2, 3, 4, 1).reshape(cout, -1).to(BF16).contiguous()
    bias = b.float().to(DEV)
    ws = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    y = Guarded((N, T, H, W, cout), BF16)
    _lib.call('og_conv3d_fwd', xr.data_ptr(), cin, k, k, k, 1, 1, 1, None, 0, packed.data_ptr(), packed.shape[1],
              bias.data_ptr(), None, None, y.ptr(), 0, N, T, H, W, cout, ws.data_ptr(), ws.numel(), None, s)
    dx = Guarded((N, T, H, W, cin), BF16)
    _lib.call('og_conv3d_dgrad', dyr.data_ptr(), cout, cout, packed.data_ptr(), packed.shape[1], 0, k, k, k, 1, 1, 1,
              dx.ptr(), 0, N, T, H, W, cin, ws.data_ptr(), ws.numel(), s)
    dw = Guarded((cout, k * k * k * cin), torch.float32, init=torch.zeros(cout, k * k * k * cin))
    db = Guarded((cout,), torch.float32, init=torch.zeros(cout))
    _lib.call('og_conv3d_wgrad_bias', dyr.data_ptr(), cout, xr.data_ptr(), cin, dw.ptr(), dw.t.shape[1], k, k, k, 1, 1,
              1, N, T, H, W, db.ptr(), cout, ws.data_ptr(), ws.numel(), s)
    torch.cuda.synchronize()
    for name, o in (('y', y), ('dx', dx), ('dw', dw), ('db', db)):
        o.check_guard(name)
    assert torch.equal(y.t, rows(y_ref).to(BF16))
    assert torch.equal(dx.t, rows(dx_ref).to(BF16))
    assert torch.equal(dw.t.double(), dw_ref.permute(0, 2, 3, 4, 1).reshape(cout, -1))
    assert torch.equal(db.t.double(), dyd.sum(dim=(0, 2, 3, 4)))


# ------------------------------------------------------------------------------------------------------------------
# blocks against the reference golden and the oracle
# ------------------------------------------------------------------------------------------------------------------
def _softmax_cancels(k):
    """A bias on every key adds q.b to all scores of a row, which the softmax cancels: the gradient of to_k.bias is zero
    in exact arithmetic, and what either side computes is rounding noise."""
    return k.endswith('to_k.bias')


def _grads(m):
    return {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}


def _ref_sd(sd):
    return {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith(('freq', 'bit_mask')))
            for k, v in sd.items()}


@GPU
@pytest.mark.parametrize('tag', CASES)
def test_block_against_reference_golden(golden, tag):
    c = golden(GOLDEN)[tag]
    m = _block(n_head=2, d_head=64, **c['kw'])
    det_weights(m)
    m.to(DEV)
    x, cond = _golden_inputs(tag, c)
    x = x.to(DEV).requires_grad_(True)
    y = m(x, cond=(None, cond.to(DEV))) if cond is not None else m(x)
    assert tuple(y.shape) == c['y_shape']
    y.backward(((2.0 / y.numel()) * y.detach().float()).to(y.dtype))
    n = c['y'].numel()
    assert rel_l2(_sample(f'stffn.y.{tag}', y, n), c['y']) < 2e-2
    assert rel_l2(_sample(f'stffn.dx.{tag}', x.grad, n), c['dx']) < 6e-2
    grads = _grads(m)
    assert sorted(grads) == c['grad_names']
    for k, got, want, norm in _golden_grads(tag, c, grads):
        assert torch.isfinite(grads[k]).all(), k
        assert _softmax_cancels(k) or rel_l2(got, want) < 8e-2, (k, rel_l2(got, want))
        assert _softmax_cancels(k) or abs(grads[k].norm().item() - norm) / norm < 8e-2, k


BLOCKS = [  # (id, n_head, d_head, kwargs, key_dim)
    ('hid4C', 2, 64, {'hid_dim': 512}, None),
    ('hid2_t1', 2, 64, {'hid_dim': (256, 384), 'transpose': True}, None),
    ('dout_t1', 2, 64, {'d_out': 256, 'transpose': True}, None),
    ('dout_hid_t1', 2, 64, {'d_out': 384, 'hid_dim': 512, 'transpose': True}, None),
    ('bias_hid_cond', 2, 64, {'bias': True, 'hid_dim': 256}, 4),
    ('bias_dout_t1', 2, 64, {'bias': True, 'd_out': 192, 'transpose': True}, None),
    ('bias_dout_hid_cond_t1', 2, 64, {'bias': True, 'd_out': 256, 'hid_dim': 256, 'transpose': True}, 4),
    ('k1', 2, 64, {'hid_dim': 512, 'kernel_size': 1}, None),
    ('k1_bias_t1', 2, 64, {'hid_dim': 256, 'kernel_size': 1, 'bias': True, 'transpose': True}, None),
    ('d128', 2, 128, {'hid_dim': 1024}, 4),
]


@GPU
@pytest.mark.parametrize('case', BLOCKS, ids=[b[0] for b in BLOCKS])
def test_block_against_oracle(case):
    tag, nh, dh, kw, cond_dim = case
    kw = dict(kw, time_attn_kw={'key_dim': cond_dim}) if cond_dim else dict(kw)
    m = _block(n_head=nh, d_head=dh, **kw)
    sd = det_weights(m)
    m.to(DEV)
    C = nh * dh
    transpose = kw.get('transpose', False)
    shape = (2, C, 16, 4, 4) if transpose else (2, 16, 4, 4, C)
    x = O.det_uniform(f'ffn.{tag}.x', shape)
    cond = O.det_uniform(f'ffn.{tag}.cond', (2, 16, cond_dim)).sign() if cond_dim else None
    xr = x.clone().requires_grad_(True)
    ref_sd = _ref_sd(sd)
    yr = FO.spacetime_attention(ref_sd, '', xr, nh, transpose, cond)
    gy = O.det_uniform(f'ffn.{tag}.gy', tuple(yr.shape), 1e-3)
    yr.backward(gy)
    xg = x.to(DEV).requires_grad_(True)
    y = m(xg, cond=(None, cond.to(DEV))) if cond_dim else m(xg)
    assert tuple(y.shape) == tuple(yr.shape)
    y.backward(gy.to(DEV).to(y.dtype))
    assert rel_l2(y.float().cpu(), yr.detach()) < 2e-2
    assert rel_l2(xg.grad.float().cpu(), xr.grad) < 6e-2
    grads = _grads(m)
    assert set(grads) == {k for k, v in ref_sd.items() if v.grad is not None}
    for k, g in grads.items():
        assert torch.isfinite(g).all(), k
        assert _softmax_cancels(k) or rel_l2(g, ref_sd[k].grad) < 8e-2, (k, rel_l2(g, ref_sd[k].grad))


@GPU
def test_gelu_passes_run_only_with_hidden_layers():
    """The entry points a block calls, forward and backward (recorded by _lib.TIMING): a default block calls exactly
    the FFN launches it always did, a block with one hidden layer adds one og_gelu_fwd and one og_gelu_bwd."""
    from open_genie_b200 import _lib
    x = torch.randn((1, 4, 4, 4, 128), device=DEV).requires_grad_(True)
    calls = {}
    for tag, kw in (('default', {}), ('hidden', {'hid_dim': 256})):
        m = _block(n_head=2, d_head=64, **kw).to(DEV)
        _lib.TIMING = []
        try:
            m(x).float().sum().backward()
            torch.cuda.synchronize()
            calls[tag] = [c[0] for c in _lib.TIMING]
        finally:
            _lib.TIMING = None
    default = ['og_gn_stats', 'og_gn_act_fwd', 'og_conv3d_fwd',
               'og_conv3d_dgrad', 'og_affine_act_bwd_reduce', 'og_conv3d_wgrad', 'og_gn_act_bwd']
    hidden = ['og_gn_stats', 'og_gn_act_fwd', 'og_conv3d_fwd', 'og_gelu_fwd', 'og_conv3d_fwd',
              'og_conv3d_dgrad', 'og_gelu_bwd', 'og_conv3d_wgrad',
              'og_conv3d_dgrad', 'og_affine_act_bwd_reduce', 'og_conv3d_wgrad', 'og_gn_act_bwd']
    for tag, want in (('default', default), ('hidden', hidden)):
        got = calls[tag]
        assert got.count('og_gn_stats') == 1, got         # the FFN's GroupNorm: its forward ends the block's forward,
        i = got.index('og_gn_stats')                      # its backward opens the block's backward
        assert got[i:i + len(want)] == want, (tag, got[i:])
        assert sum(n.startswith('og_gelu') for n in got) == (2 if tag == 'hidden' else 0)


# ------------------------------------------------------------------------------------------------------------------
# models, CUDA graphs, zero arena
# ------------------------------------------------------------------------------------------------------------------
def _dyn_inputs(T, hw, vocab, act_vocab, tag):
    shape = (2, T, hw, hw)
    u = O.det_uniform(f'{tag}.tokens', shape) / (3 ** 0.5)
    tokens = ((u + 1) * 0.5 * vocab).long().clamp(0, vocab - 1)
    ua = O.det_uniform(f'{tag}.act', shape[:2]) / (3 ** 0.5)
    act = ((ua + 1) * 0.5 * act_vocab).long().clamp(0, act_vocab - 1)
    mask = O.det_uniform(f'{tag}.mask', shape) / (3 ** 0.5) < 0.5
    return tokens, act, mask


@GPU
@pytest.mark.parametrize('nh,hid,T,hw', [(2, 512, 4, 8), (8, 2048, 2, 4)])
def test_dynamics_with_hidden_ffn_against_oracle(nh, hid, T, hw):
    """The second case is DynamicsModel((('space-time_attn', {'n_rep': 2, 'n_head': 8, 'd_head': 64,
    'hid_dim': 2048}),), 1024, 8, 512), trained for one step."""
    import open_genie_b200 as og
    desc = (('space-time_attn', {'n_rep': 2, 'n_head': nh, 'd_head': 64, 'hid_dim': hid}),)
    vocab, act_vocab, embed = (64, 16, 128) if nh == 2 else (1024, 8, 512)
    dm = og.DynamicsModel(desc, vocab, act_vocab, embed)
    sd = det_weights(dm)
    dm.to(DEV)
    tokens, act, mask = _dyn_inputs(T, hw, vocab, act_vocab, f'ffn.dyn.{nh}')
    ref_sd = _ref_sd(sd)
    with FO.blueprints():
        ref_loss = O.dynamics_loss(ref_sd, desc, tokens, act, mask)
    ref_loss.backward()
    loss = dm.compute_loss(tokens.to(DEV), act.to(DEV), mask=mask.to(DEV))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) / ref_loss.item() < 2e-2
    grads = _grads(dm)
    assert any('.ffn.1.net.2.0.weight' in k for k in grads)
    for k, g in grads.items():
        r = ref_sd[k].grad
        assert r is not None, k
        assert rel_l2(g, r) < 0.1, (k, rel_l2(g, r))
    opt = og.FusedAdamW(dm.parameters(), lr=1e-3)
    before = {k: p.detach().clone() for k, p in dm.named_parameters()}
    opt.step()
    torch.cuda.synchronize()
    assert all(not torch.equal(p.detach(), before[k]) for k, p in dm.named_parameters() if p.grad is not None)


@GPU
def test_latent_action_with_hidden_ffn_against_oracle():
    import open_genie_b200 as og
    wide = lambda bp: tuple((n, {**kw, 'hid_dim': 256} if n == 'space-time_attn' else kw) for n, kw in bp)
    enc, dec = wide(fx.MINI_ACT_ENC), wide(fx.MINI_ACT_DEC)
    la = og.LatentAction(enc, dec, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                         inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:])
    sd = det_weights(la)
    assert 'enc_layers.0.ffn.1.net.2.0.weight' in sd and 'dec_layers.0.ffn.1.net.2.0.weight' in sd
    la.to(DEV).train()
    video = O.det_uniform('ffn.action.video', fx.MINI_ACT_VIDEO_SHAPE)
    ref_sd = _ref_sd(sd)
    with FO.blueprints():
        _, ref_loss, (ref_rec, _), _ = O.latent_action_forward(ref_sd, enc, dec, video, fx.MINI_ACT_D_CODEBOOK)
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


def _graph_block():
    m = _block(n_head=2, d_head=64, hid_dim=256, d_out=192, bias=True, transpose=True)
    det_weights(m)
    return m.to(DEV)


@GPU
def test_block_cuda_graph_replay_matches_eager():
    m = _graph_block()
    shape = (2, 128, 16, 4, 4)
    x = O.det_uniform('ffn.graph.x', shape).to(DEV).requires_grad_(True)
    gy = O.det_uniform('ffn.graph.gy', (2, 192, 16, 4, 4), 1e-3).to(DEV)

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
    assert set(g_e) == {k for k, p in m.named_parameters() if p.grad is not None}
    for k, p in m.named_parameters():
        if k in g_e:
            assert rel_l2(p.grad.float().cpu(), g_e[k].float().cpu()) < 8e-2, k


@GPU
def test_zero_arena_gives_the_same_gradients():
    """Weight, bias and shortcut gradients taken from the step's zero arena (og.enable_zero_arena) equal those taken
    from torch.zeros."""
    import open_genie_b200 as og
    from open_genie_b200 import ops
    m = _graph_block()
    x = O.det_uniform('ffn.arena.x', (2, 128, 16, 4, 4)).to(DEV).requires_grad_(True)
    gy = O.det_uniform('ffn.arena.gy', (2, 192, 16, 4, 4), 1e-3).to(DEV)

    def step():
        x.grad = None
        m.zero_grad(set_to_none=True)
        m(x).backward(gy.to(BF16))
        torch.cuda.synchronize()
        return x.grad.clone(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    dx0, g0 = step()
    og.enable_zero_arena(True)
    try:
        for _ in range(2):                      # the second step runs on a recycled (re-zeroed) arena
            ops.mark_step()
            dx1, g1 = step()
            assert ops.ZERO_ARENA.bytes_in_use() > 0
            # the same kernels on the same inputs; the GroupNorm statistics are fp64 atomic sums, whose order (and so
            # the last bits of what follows) is not fixed from run to run
            assert rel_l2(dx1.float().cpu(), dx0.float().cpu()) < 1e-3
            for k in g0:
                assert rel_l2(g1[k].cpu(), g0[k].cpu()) < 1e-3, k
    finally:
        og.enable_zero_arena(False)
        ops.mark_step()
