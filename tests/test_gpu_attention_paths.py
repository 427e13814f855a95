"""Every dispatch path of the attention kernels against an explicit float64 reference, element by element.

Paths covered: the mma.sync temporal kernels (d_head 64, T <= 16), the per-lane temporal kernels (`<64>` for T in
17..32, `<32>` for every T, two tasks per warp when T <= 16), the wgmma flash attention at ragged S and at S = 4096,
the RoPE+LayerNorm backward (vectorised and generic kernel), and the composed autograd functions of ops.py.

Every tolerance is a per-element worst-case bound built from the rounding points of the path under test
(`attn_err`, `rope_ln_bwd_expect`). The `test_tolerance(s)_reject_*` tests run on the CPU and show that each bound
still rejects the mistakes it exists to catch.
"""
import pytest
import torch

from helpers import Guarded
from oracle import genie_oracle as O

GPU = pytest.mark.gpu
DEV = 'cuda'
BF16, F32T = torch.bfloat16, torch.float32

# Rounding model. U is the unit roundoff of bf16 (8 significant bits): |bf16(x) - x| <= U |x|. F32 is one fp32 ulp;
# tensor-core and fma sums may truncate rather than round, so a sum of n terms is taken to be within n * F32 of the
# exact sum, relative to the sum of the terms' magnitudes (`gam`).
U = 2.0 ** -8
F32 = 2.0 ** -23
# fp32 slack of the RoPE+LayerNorm passes, relative to the magnitudes involved: covers gam(n) for the C <= 1024 channel
# sums and a few hundred rows of dgamma / dbeta, sincosf's 2-ulp error and the fp32 mean / variance.
F_LN = 2.0 ** -12
SLACK = 1.02    # second-order terms (an error that is itself rounded, U * err) are folded into this factor
# Absolute floor of every bound. Below fp32's normal range (2^-126) there is no relative precision: exp2.approx flushes
# such probabilities to zero, and a flushed P entry moves an output by less than 2^-126 * sum |v| << 2^-100 here.
# (Large scores put many dK / dS entries at 1e-40.)
TINY = 2.0 ** -100


def gam(n):
    return n * F32


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
def attn_ref(q, k, v, scale, causal=False, do=None, diag=0):
    """Explicit attention on [..., S, d] float64 tensors (batch dims broadcast): scores, mask, softmax, output, log-sum-
    exp, and dQ / dK / dV in closed form. `diag` shifts the causal diagonal (only the sensitivity test changes it)."""
    s = scale * (q @ k.transpose(-1, -2))
    if causal:
        keep = torch.ones(s.shape[-2:], dtype=torch.bool, device=s.device).tril(diag)
        s = s.masked_fill(~keep, float('-inf'))
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    r = {'p': p, 'o': p @ v, 'lse': (m + l.log()).squeeze(-1)}
    if do is not None:
        dp = do @ v.transpose(-1, -2)
        ds = p * (dp - (p * dp).sum(-1, keepdim=True))
        r.update(ds=ds, dq=scale * (ds @ k), dk=scale * (ds.transpose(-1, -2) @ q), dv=p.transpose(-1, -2) @ do)
    return r


def attn_err(q, k, v, r, scale, p_bf16, do=None, delta_from_bf16_o=False):
    """Worst-case |kernel - r| per element before each output's own bf16 rounding, for kernels fed these exact inputs.

    fp32 parts, common to every path:
      * a score is a d-term fp32 dot product: |err| <= gam(2d) * scale * (|q| . |k|), so a row of P (numerator and row
        sum) is off by at most twice the row's largest score error, relatively; `exp2.approx` and the saved log-sum-exp
        add gam(4) * (1 + |lse|). Together with the n-term sums over keys this is the relative slack `rho`.
    Rounding points:
      * p_bf16 (mma.sync temporal, flash): P is rounded to bf16 before P V and P^T dO, and dS before dS K and dS^T Q:
        each product is then off by U * (|P| |V|), U * (|dS| |K|), ... on top of rho.
      * per-lane temporal: P and dS stay fp32, only rho applies.
      * flash backward (delta_from_bf16_o): delta = rowsum(dO * O) uses the stored bf16 output, whose error is the
        forward bound plus U |O|; that error times P enters dS.
    """
    aq, ak, av = q.abs(), k.abs(), v.abs()
    p = r['p']
    g = gam(k.shape[-2] + 128)
    es = (gam(2 * q.shape[-1]) * scale) * (aq @ ak.transpose(-1, -2))
    es = torch.where(p > 0, es, torch.zeros_like(es)).amax(-1, keepdim=True)
    rho = g + 2 * es + gam(4) * (1 + r['lse'].abs()).unsqueeze(-1)
    up = U if p_bf16 else 0.0
    err = {'o': (up + rho) * (p @ av), 'lse': rho.squeeze(-1)}
    if do is None:
        return err
    ado = do.abs()
    dp_mag = ado @ av.transpose(-1, -2)
    ed = (rho + g) * (p * dp_mag).sum(-1, keepdim=True)
    if delta_from_bf16_o:
        ed = ed + (ado * (err['o'] + U * r['o'].abs())).sum(-1, keepdim=True)
    ads = r['ds'].abs()
    eds = (up + rho + g) * ads + p * (ed + g * dp_mag)
    err['dq'] = scale * (eds @ ak)
    err['dk'] = scale * (eds.transpose(-1, -2) @ aq)
    err['dv'] = (up + rho + g) * (p.transpose(-1, -2) @ ado)
    return err


def bf16_tol(err, ref):
    """Bound of a bf16 output: the fp32 result's bound plus the final rounding."""
    return SLACK * (err + U * ref.abs())


# temporal layouts: q / out rows ((b*T + t)*P + p) of C = nh*d channels <-> [B, P, nh, T, d] sequences
def _tseq(x, nh):
    B, T, P, C = x.shape
    return x.view(B, T, P, nh, C // nh).permute(0, 2, 3, 1, 4)


def _tunseq(y):
    B, P, nh, T, d = y.shape
    return y.permute(0, 3, 1, 2, 4).reshape(B, T, P, nh * d)


def _kvseq(k, nh):      # broadcast K / V [B, T, C] -> [B, 1, nh, T, d]
    B, T, C = k.shape
    return k.view(B, T, nh, C // nh).permute(0, 2, 1, 3)[:, None]


def _kvsum(y):          # per-pixel [B, P, nh, T, d] -> summed over the pixels, [B, T, C]
    B, P, nh, T, d = y.shape
    return y.sum(1).permute(0, 2, 1, 3).reshape(B, T, nh * d)


def temporal_uses_mma(d, T):
    """The dispatch rule of og_temporal_attn_fwd / bwd; `test_dispatch_kernel_names` pins it to the kernels."""
    return d == 64 and T <= 16


def temporal_expect(q, k, v, do, res, nh, scale, bcast, dk_init=None, dv_init=None):
    """{output: (reference, tolerance)} of og_temporal_attn_fwd / bwd on these bf16 inputs, in the kernels' layouts.
    q, do, res: [B, T, P, C]; k, v: the same (bcast = 0) or [B, T, C] (bcast = 1)."""
    B, T, P, C = q.shape
    mma = temporal_uses_mma(C // nh, T)
    f = lambda t: t.double()
    qs, dos = _tseq(f(q), nh), _tseq(f(do), nh)
    ks, vs = (_kvseq(f(k), nh), _kvseq(f(v), nh)) if bcast else (_tseq(f(k), nh), _tseq(f(v), nh))
    r = attn_ref(qs, ks, vs, scale, causal=True, do=dos)
    e = attn_err(qs, ks, vs, r, scale, p_bf16=mma, do=dos)
    o, eo = _tunseq(r['o']), _tunseq(e['o'])
    out = {'out': (o, bf16_tol(eo, o))}
    if res is not None:
        orr = o + f(res)
        # The mma.sync kernel rounds the attention output to bf16 before it adds the residual (frags_to_tile, then
        # tile_to_global): two roundings, U |o| + U |o + res|. The per-lane kernels add in fp32 and round once.
        tol = eo + U * orr.abs() + (U * o.abs() if mma else 0)
        out['out_res'] = (orr, SLACK * tol)
    out['dq'] = (_tunseq(r['dq']), bf16_tol(_tunseq(e['dq']), _tunseq(r['dq'])))
    if bcast:
        # fp32 accumulators, ACCUMULATED into the caller's values: per-pixel bounds add up, plus the fp32 sum over
        # the pixels and the caller's value
        for name, init in (('dk', dk_init), ('dv', dv_init)):
            init = torch.zeros_like(f(k)) if init is None else f(init)
            ref = init + _kvsum(r[name])
            tol = _kvsum(e[name]) + gam(P + 2) * (init.abs() + _kvsum(r[name].abs()))
            out[name + '_bcast'] = (ref, SLACK * tol)
    else:
        for name in ('dk', 'dv'):
            out[name] = (_tunseq(r[name]), bf16_tol(_tunseq(e[name]), _tunseq(r[name])))
    return out


def flash_expect(q, k, v, do, res, nh, scale):
    """{output: (reference, tolerance)} of og_flash_attn_fwd / bwd on these bf16 [nseq, S, C] inputs."""
    nseq, S, C = q.shape
    sp = lambda t: t.double().view(nseq, S, nh, C // nh).transpose(1, 2)
    un = lambda t: t.transpose(1, 2).reshape(nseq, S, C)
    qs, ks, vs, dos = sp(q), sp(k), sp(v), sp(do)
    r = attn_ref(qs, ks, vs, scale, do=dos)
    e = attn_err(qs, ks, vs, r, scale, p_bf16=True, do=dos, delta_from_bf16_o=True)
    out = {name: (un(r[name]), bf16_tol(un(e[name]), un(r[name]))) for name in ('o', 'dq', 'dk', 'dv')}
    out['out'] = out.pop('o')
    out['lse'] = (r['lse'], SLACK * e['lse'])
    if res is not None:
        orr = un(r['o']) + res.double()
        out['out_res'] = (orr, SLACK * (un(e['o']) + U * orr.abs()))
    return out


def check(name, got, ref, tol):
    got = got.double().to(ref.device)
    assert got.shape == ref.shape, f'{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
    tol = tol + TINY
    bad = ~(err <= tol)    # NaN (an element never written) is bad too
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        ratio = (err / tol.clamp_min(1e-300)).flatten().nan_to_num(float('inf')).max().item()
        raise AssertionError(
            f'{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound, worst err/tol {ratio:.3g}; first at '
            f'flat index {i} (of shape {tuple(ref.shape)}): got {got.flatten()[i].item():.6g}, '
            f'ref {ref.flatten()[i].item():.6g}, tol {tol.flatten()[i].item():.3g}')


def check_all(got, expect):
    for name, t in got.items():
        check(name, t, *expect[name])


# RoPE + LayerNorm
def rope_ln_ref(x, pos, freq, gamma, beta, eps=1e-5):
    """float64 LayerNorm(RoPE(x)) of rows x [R, C] at positions pos [R]. The angle is the fp32 product pos * freq[i],
    as the reference module computes it (attention.py:48-94)."""
    ang = (pos.float()[:, None] * freq.float()[None, :].to(pos.device)).double()
    c, s = ang.cos(), ang.sin()
    x0, x1 = x[:, 0::2], x[:, 1::2]
    r = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), -1).flatten(1)
    mu = r.mean(-1, keepdim=True)
    rstd = ((r - mu).pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    xh = (r - mu) * rstd
    return {'c': c, 's': s, 'xh': xh, 'rstd': rstd, 'y': xh * gamma.double() + beta.double()}


def _rot_t(d, st, absolute=False):
    """R^T d, the transpose of the RoPE rotation; with absolute=True the same map on |cos|, |sin| (error propagation)."""
    c, s = (st['c'].abs(), st['s'].abs()) if absolute else (st['c'], st['s'])
    d0, d1 = d[:, 0::2], d[:, 1::2]
    return torch.stack((d0 * c + d1 * s, (d0 * s if absolute else -d0 * s) + d1 * c), -1).flatten(1)


def _ln_bwd(st, g, gamma, absolute=False):
    gh = g * (gamma.double().abs() if absolute else gamma.double())
    xh = st['xh'].abs() if absolute else st['xh']
    sign = 1 if absolute else -1
    return st['rstd'] * (gh + sign * gh.mean(-1, keepdim=True) + sign * xh * (gh * xh).mean(-1, keepdim=True))


def rope_ln_bwd_expect(st, g, gamma, add, eg=None, dg_init=None, db_init=None):
    """{output: (reference, tolerance)} of og_rope_ln_bwd for the gradient g = g0 + g1 + g2 (float64) and `add`.
    eg: per-element bound of g itself when it is not exact (the composed functions' bf16 attention gradients): it is
    propagated through |d dx / d g|. dx is bf16; dgamma / dbeta fp32, accumulated into dg_init / db_init."""
    dx = _rot_t(_ln_bwd(st, g, gamma), st) + add
    mag = _rot_t(_ln_bwd(st, g.abs(), gamma, True), st, True) + add.abs()
    ex = F_LN * mag
    ag, axh = g.abs(), st['xh'].abs()
    egam, ebet = F_LN * (ag * (axh + 1)).sum(0), F_LN * ag.sum(0)
    if eg is not None:
        ex = ex + _rot_t(_ln_bwd(st, eg, gamma, True), st, True)
        egam, ebet = egam + (eg * axh).sum(0), ebet + eg.sum(0)
    dgam, dbet = (g * st['xh']).sum(0), g.sum(0)
    if dg_init is not None:
        dgam, dbet = dgam + dg_init.double(), dbet + db_init.double()
        egam, ebet = egam + F_LN * dg_init.double().abs(), ebet + F_LN * db_init.double().abs()
    return {'dx': (dx, bf16_tol(ex, dx)), 'dgamma': (dgam, SLACK * egam), 'dbeta': (dbet, SLACK * ebet)}


# ------------------------------------------------------------------------------------------------------------------
# CPU: the tolerances reject the mistakes they exist to catch
# ------------------------------------------------------------------------------------------------------------------
def _cpu_rand(shape, seed, amp=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * amp).to(BF16)


def _bf(t):
    return t.to(BF16)


def _rejects(got, expect):
    with pytest.raises(AssertionError):
        check_all(got, expect)


@pytest.mark.parametrize('d,T', [(64, 8), (64, 24), (32, 8)])
def test_tolerances_reject_plausible_bugs_temporal(d, T):
    """A kernel that is exactly right (the reference rounded to bf16) passes; each mutation is rejected. Both rounding
    models are exercised: d = 64, T <= 16 is the mma.sync path (P, dS in bf16), the others the per-lane path."""
    B, P, nh = 2, 3, 2
    C, scale = nh * d, nh * d ** -0.5
    assert scale != 1.0
    q, k, v, do, res = (_cpu_rand((B, T, P, C), 100 + i, 1.0) for i in range(5))
    ex = temporal_expect(q, k, v, do, res, nh, scale, bcast=False)
    exact = {n: _bf(t[0]) for n, t in ex.items()}
    check_all(exact, ex)
    f = lambda t: t.double()
    qs, ks, vs, dos = _tseq(f(q), nh), _tseq(f(k), nh), _tseq(f(v), nh), _tseq(f(do), nh)

    def variant(**kw):
        a = dict(scale=scale, causal=True, do=dos)
        a.update(kw)
        return attn_ref(qs, ks, vs, **a)
    # the causal mask off by one
    _rejects({'out': _bf(_tunseq(variant(diag=1)['o']))}, ex)
    _rejects({'dq': _bf(_tunseq(variant(diag=1)['dq']))}, ex)
    # dk and dv swapped
    _rejects({'dk': exact['dv'], 'dv': exact['dk']}, ex)
    # the residual omitted
    _rejects({'out_res': exact['out']}, ex)
    # the softmax scale applied twice
    _rejects({'out': _bf(_tunseq(variant(scale=scale * scale)['o']))}, ex)
    _rejects({'dq': _bf(_tunseq(variant(scale=scale * scale)['dq']))}, ex)
    # one head's columns taken from the neighbouring head
    for name in ('out', 'dk'):
        bad = exact[name].clone()
        bad[..., :d] = exact[name][..., d:2 * d]
        _rejects({name: bad}, ex)
    # broadcast K / V: the caller's values overwritten instead of accumulated, and one (b, h) flushed to the next b
    kb, vb = _cpu_rand((B, T, C), 110, 1.0), _cpu_rand((B, T, C), 111, 1.0)
    init = _cpu_rand((B, T, C), 112, 1.0).float()
    exb = temporal_expect(q, kb, vb, do, None, nh, scale, bcast=True, dk_init=init, dv_init=init)
    right = exb['dk_bcast'][0].float()
    check_all({'dk_bcast': right}, exb)
    _rejects({'dk_bcast': right - init}, exb)
    _rejects({'dk_bcast': right.flip(0)}, exb)


def test_tolerances_reject_plausible_bugs_flash():
    nseq, S, nh = 2, 100, 2
    C, scale = 64 * nh, nh * 64 ** -0.5
    q, k, v, do, res = (_cpu_rand((nseq, S, C), 200 + i, 1.0) for i in range(5))
    ex = flash_expect(q, k, v, do, res, nh, scale)
    exact = {n: (t[0].float() if n == 'lse' else _bf(t[0])) for n, t in ex.items()}
    check_all(exact, ex)
    sp = lambda t: t.double().view(nseq, S, nh, 64).transpose(1, 2)
    un = lambda t: t.transpose(1, 2).reshape(nseq, S, C)
    qs, ks, vs, dos = sp(q), sp(k), sp(v), sp(do)
    # the last partial key tile (keys 64..99) dropped
    cut = attn_ref(qs, ks[..., :64, :], vs[..., :64, :], scale, do=dos)
    _rejects({'out': _bf(un(cut['o']))}, ex)
    _rejects({'lse': cut['lse'].float()}, ex)
    _rejects({'dq': _bf(un(cut['dq']))}, ex)
    # dk and dv swapped; the residual omitted; the scale applied twice; a head shifted
    _rejects({'dk': exact['dv'], 'dv': exact['dk']}, ex)
    _rejects({'out_res': exact['out']}, ex)
    twice = attn_ref(qs, ks, vs, scale * scale, do=dos)
    _rejects({'out': _bf(un(twice['o']))}, ex)
    _rejects({'dk': _bf(un(twice['dk']))}, ex)
    bad = exact['out'].clone()
    bad[..., 64:] = exact['out'][..., :64]
    _rejects({'out': bad}, ex)


def test_tolerance_rejects_wrong_rope_ln_backward():
    rows, C = 40, 128
    x = _cpu_rand((rows, C), 300).double()
    pos = torch.arange(rows) % 5
    freq = O.rope_freq(C, '1d')
    gamma, beta = 1 + 0.2 * torch.randn(C, generator=torch.Generator().manual_seed(1)), torch.zeros(C)
    st = rope_ln_ref(x, pos, freq, gamma, beta)
    g, add = _cpu_rand((rows, C), 301).double(), _cpu_rand((rows, C), 302).double()
    ex = rope_ln_bwd_expect(st, g, gamma, add)
    check_all({'dx': _bf(ex['dx'][0]), 'dgamma': ex['dgamma'][0].float()}, ex)
    _rejects({'dx': _bf(ex['dx'][0] - add)}, ex)                                           # `add` dropped
    _rejects({'dx': _bf(_rot_t(_ln_bwd(st, g, gamma), {'c': st['c'], 's': -st['s']}) + add)}, ex)  # R instead of R^T
    _rejects({'dgamma': (ex['dgamma'][0] - (g[-1] * st['xh'][-1])).float()}, ex)          # the last row dropped


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation of the attention entry points (no device needed)
# ------------------------------------------------------------------------------------------------------------------
def test_attention_argument_validation_returns_status_codes():
    import ctypes
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    # flash backward: empty problems and a non-positive scale, as the forward rejects them
    for nseq, S, scale in ((1, 0, 1.0), (0, 64, 1.0), (1, 64, 0.0), (1, 64, -1.0)):
        rc = lib.og_flash_attn_bwd(p, p, p, p, p, p, p, p, p, p, nseq, S, 64, 1, scale, None)
        assert rc == -1, (nseq, S, scale, rc)
        rc = lib.og_flash_attn_fwd(p, p, p, p, None, None, p, nseq, S, 64, 1, scale, None)
        assert rc == -1, (nseq, S, scale, rc)
    assert b'scale' in lib.og_last_error()
    rc = lib.og_flash_attn_bwd(p, p, p, p, p, p, p, p, p, p, 1, 64, 96, 2, 1.0, None)     # d_head 48
    assert rc == -1 and b'd_head = 64' in lib.og_last_error()
    # temporal: B and P must be positive; d_head must be 32 or 64
    for B, P in ((0, 4), (1, 0), (-1, 4)):
        assert lib.og_temporal_attn_fwd(p, p, p, None, p, B, 8, P, 128, 2, 1.0, 0, None) == -1
        assert b'empty problem' in lib.og_last_error()
        assert lib.og_temporal_attn_bwd(p, p, p, p, p, p, p, None, None, B, 8, P, 128, 2, 1.0, 0, None) == -1
        assert b'empty problem' in lib.og_last_error()
    assert lib.og_temporal_attn_fwd(p, p, p, None, p, 1, 8, 4, 96, 2, 1.0, 0, None) == -2
    assert b'd_head=48' in lib.og_last_error()
    assert lib.og_temporal_attn_bwd(p, p, p, p, p, p, p, None, None, 1, 8, 4, 96, 2, 1.0, 0, None) == -2
    assert b'd_head=48' in lib.og_last_error()
    assert lib.og_temporal_attn_fwd(p, p, p, None, p, 1, 33, 4, 128, 2, 1.0, 0, None) == -1


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _rand(shape, seed, amp=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * amp).to(BF16)


def _ptr(t):
    return None if t is None else t.data_ptr()


def temporal_run(B, T, P, nh, d, bcast, seed, amp=1.0, aliased=False, do_mask=None, check_guards=True):
    """Runs og_temporal_attn_fwd (without and with a residual) and og_temporal_attn_bwd on guarded outputs and checks
    every output against `temporal_expect`. The broadcast K/V gradients start from non-zero values."""
    C, scale = nh * d, nh * d ** -0.5
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
    out, out_res, dq = (Guarded(q.shape, BF16, G) for _ in range(3))
    _call('og_temporal_attn_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), None, out.ptr(), B, T, P, C, nh, scale,
          int(bcast))
    _call('og_temporal_attn_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), res.data_ptr(), out_res.ptr(), B, T, P, C,
          nh, scale, int(bcast))
    outs = {'out': out, 'out_res': out_res, 'dq': dq}
    dk_init = dv_init = None
    if bcast:
        dk_init, dv_init = _rand((B, T, C), seed + 5).float(), _rand((B, T, C), seed + 6).float()
        outs['dk_bcast'] = Guarded((B, T, C), F32T, G, dk_init)
        outs['dv_bcast'] = Guarded((B, T, C), F32T, G, dv_init)
        _call('og_temporal_attn_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), do.data_ptr(), dq.ptr(), None, None,
              outs['dk_bcast'].ptr(), outs['dv_bcast'].ptr(), B, T, P, C, nh, scale, 1)
    else:
        outs['dk'], outs['dv'] = Guarded(q.shape, BF16, G), Guarded(q.shape, BF16, G)
        _call('og_temporal_attn_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), do.data_ptr(), dq.ptr(),
              outs['dk'].ptr(), outs['dv'].ptr(), None, None, B, T, P, C, nh, scale, 0)
    torch.cuda.synchronize()
    ex = temporal_expect(q, k, v, do, res, nh, scale, bcast, dk_init, dv_init)
    check_all({n: o.t for n, o in outs.items()}, ex)
    if check_guards:
        for n, o in outs.items():
            o.check_guard(n)
    inputs = {'q': q, 'k': k, 'v': v, 'do': do, 'res': res, 'dk_init': dk_init, 'dv_init': dv_init}
    return inputs, {n: o.t for n, o in outs.items()}


# ------------------------------------------------------------------------------------------------------------------
# temporal attention: mma.sync path
# ------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('nh', [1, 2, 8])
@pytest.mark.parametrize('T', [1, 2, 7, 15, 16])
def test_temporal_mma_path(T, nh, bcast):
    assert temporal_uses_mma(64, T)
    temporal_run(B=2, T=T, P=24, nh=nh, d=64, bcast=bcast, seed=1000 + 10 * T + nh)


@GPU
@pytest.mark.parametrize('T,d', [(16, 64), (5, 64), (24, 64), (16, 32)])
def test_temporal_aliased_product_call(T, d):
    """q = k = v, as _TimeAttnFn makes the call (ops.py:979, 1003): dq, dk and dv are the three partial gradients of the
    same tensor, each checked on its own."""
    temporal_run(B=2, T=T, P=20, nh=2, d=d, bcast=0, seed=2000 + T + d, aliased=True)


# ------------------------------------------------------------------------------------------------------------------
# temporal attention: per-lane path. B*P*nh = 21 tasks: with two tasks per warp (T <= 16) the last warp step is odd.
# ------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize('bcast', [0, 1])
@pytest.mark.parametrize('d,T', [(64, 17), (64, 24), (64, 32), (32, 1), (32, 5), (32, 16), (32, 17), (32, 32)])
def test_temporal_per_lane_path(d, T, bcast):
    assert not temporal_uses_mma(d, T)
    temporal_run(B=1, T=T, P=7, nh=3, d=d, bcast=bcast, seed=3000 + 10 * T + d)


# ------------------------------------------------------------------------------------------------------------------
# temporal attention: many tasks per warp, warp ranges that straddle (b, h) boundaries, large scores
# ------------------------------------------------------------------------------------------------------------------
def _bwd_warp_ranges(ntask, mma, tpw):
    """The backward launchers' static work split (attention_rows.cu, temporal_attn_mma.cu): [begin, end) per warp."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = min((ntask + 3) // 4, sms * (4 if mma else 8)) * 4
    per = -(-ntask // warps)
    per = -(-per // tpw) * tpw
    return [(w * per, min(w * per + per, ntask)) for w in range(warps) if w * per < ntask]


@GPU
@pytest.mark.parametrize('bcast', [0, 1])
def test_temporal_mma_many_tasks_per_warp(bcast):
    """The model's shape: T = 16, P = 64 x 64 pixels, 8 heads. 32768 tasks: each warp runs several in a row."""
    B, T, P, nh = 1, 16, 4096, 8
    ranges = _bwd_warp_ranges(B * P * nh, True, 1)
    assert max(e - b for b, e in ranges) >= 4
    temporal_run(B, T, P, nh, 64, bcast, seed=4000 + bcast)


@GPU
@pytest.mark.parametrize('d,T', [(64, 16), (64, 24), (32, 16)])
def test_temporal_bcast_gradient_straddles_bh(d, T):
    """kv_bcast = 1 with P = 999: warp ranges cross (b, h) boundaries, so a warp flushes its K/V gradient registers
    mid-range and starts a new (b, h). A second backward pass has dO non-zero only on the first two and last two
    pixels of every (b, h) (the tasks at the range edges), so the sum over pixels has few terms and a lost or
    misrouted contribution is far outside the bound even on the mma.sync path, whose per-pixel bound is U-sized."""
    B, P, nh = 2, 999, 4
    mma = temporal_uses_mma(d, T)
    tpw = 1 if mma or T > 16 else 2
    ranges = _bwd_warp_ranges(B * P * nh, mma, tpw)
    straddle = [r for r in ranges if r[0] // P != (r[1] - 1) // P]
    assert len(straddle) >= B * nh // 2, 'the shape no longer makes warp ranges cross (b, h) boundaries'
    temporal_run(B, T, P, nh, d, 1, seed=5000 + T + d)
    edge = torch.zeros(P, device=DEV, dtype=BF16)
    edge[[0, 1, P - 2, P - 1]] = 1
    temporal_run(B, T, P, nh, d, 1, seed=5100 + T + d, do_mask=edge.view(1, 1, P, 1), check_guards=False)


@GPU
@pytest.mark.parametrize('d,T', [(64, 16), (64, 9), (64, 32), (32, 16)])
def test_temporal_large_scores(d, T):
    """|scale q.k| around 40 and beyond 89 in places: without the row maximum subtracted first, exp overflows fp32."""
    B, P, nh = 2, 16, 2
    inp, _ = temporal_run(B, T, P, nh, d, 0, seed=6000 + T + d, amp=4.5)
    s = (nh * d ** -0.5) * (_tseq(inp['q'].float(), nh) @ _tseq(inp['k'].float(), nh).transpose(-1, -2))
    s = s.tril()    # the scores the causal mask keeps
    assert s.abs().amax().item() > 89, 'scores too small to overflow exp without the max subtraction'


@GPU
@pytest.mark.parametrize('d,bcast', [(64, 0), (64, 1), (32, 0), (32, 1)])
def test_temporal_T1_is_exact(d, bcast):
    """One time step: the softmax is exactly 1, so out = v[0] (+ residual, rounded once), dq = dk = 0, dv = dout."""
    B, T, P, nh = 2, 1, 9, 2
    inp, got = temporal_run(B, T, P, nh, d, bcast, seed=7000 + d + bcast)
    v = inp['v']
    vb = v[:, :, None].expand(B, T, P, nh * d) if bcast else v
    assert torch.equal(got['out'], vb)
    assert torch.equal(got['out_res'], (vb.float() + inp['res'].float()).to(BF16))
    assert torch.equal(got['dq'], torch.zeros_like(got['dq']))
    if bcast:   # dk adds exact zeros to the caller's values; dv (a sum over pixels) is checked by temporal_run
        assert torch.equal(got['dk_bcast'], inp['dk_init'])
    else:
        assert torch.equal(got['dk'], torch.zeros_like(got['dk']))
        assert torch.equal(got['dv'], inp['do'])


@GPU
@pytest.mark.parametrize('d,T,bcast', [(64, 16, 0), (64, 16, 1), (64, 11, 0), (64, 24, 0), (32, 16, 1), (32, 29, 0)])
def test_temporal_causality_is_exact(d, T, bcast):
    """Changing K/V rows t' > t0 must leave output rows <= t0 bit-identical (and change the later ones)."""
    B, P, nh = 2, 10, 2
    C, scale = nh * d, nh * d ** -0.5
    q = _rand((B, T, P, C), 8000)
    kvshape = (B, T, C) if bcast else (B, T, P, C)
    k, v = _rand(kvshape, 8001), _rand(kvshape, 8002)
    t0 = T // 2
    k2, v2 = k.clone(), v.clone()
    k2[:, t0 + 1:] = _rand(k2[:, t0 + 1:].shape, 8003, 3.0)
    v2[:, t0 + 1:] = _rand(v2[:, t0 + 1:].shape, 8004, 3.0)
    outs = []
    for kk, vv in ((k, v), (k2, v2)):
        o = torch.empty_like(q)
        _call('og_temporal_attn_fwd', q.data_ptr(), kk.data_ptr(), vv.data_ptr(), None, o.data_ptr(), B, T, P, C, nh,
              scale, bcast)
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][:, :t0 + 1], outs[1][:, :t0 + 1])
    assert not torch.equal(outs[0][:, t0 + 1:], outs[1][:, t0 + 1:])


# ------------------------------------------------------------------------------------------------------------------
# flash attention
# ------------------------------------------------------------------------------------------------------------------
def flash_run(nseq, S, nh, seed, amp=0.5, aliased=False):
    C, scale = 64 * nh, nh * 64 ** -0.5
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
@pytest.mark.parametrize('S', [1, 16, 63, 65, 100, 200, 257])
def test_flash_ragged_S(S):
    """S not a multiple of the 64-row tile: the forward's last-key-tile mask, the backward's row / column masks and the
    row drop of the stores; lse against the float64 log-sum-exp; out_res = bf16(o + res) with out still written."""
    flash_run(nseq=3, S=S, nh=2, seed=9000 + S)


@GPU
def test_flash_full_size_frame():
    """S = 4096: a 64 x 64 frame, the product's largest sequence."""
    flash_run(nseq=1, S=4096, nh=2, seed=9500)


@GPU
@pytest.mark.parametrize('S,nh', [(100, 2), (256, 4)])
def test_flash_aliased_product_call(S, nh):
    """q = k = v with a residual, as _SpaceAttnFn makes the call (ops.py:930, 946): dq, dk, dv each against float64."""
    flash_run(nseq=2, S=S, nh=nh, seed=9700 + S, aliased=True)


# ------------------------------------------------------------------------------------------------------------------
# RoPE + LayerNorm backward with every gradient input, vectorised and generic kernels
# ------------------------------------------------------------------------------------------------------------------
def _rope_ln_inputs(C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    gamma = 1 + 0.2 * torch.randn(C, generator=g, device=DEV)
    beta = 0.2 * torch.randn(C, generator=g, device=DEV)
    return gamma, beta


def _rope_ln_bwd_call(x, freq, gamma, g0, g1, g2, add, dg0, db0, pos_div, pos_mod, offset):
    """og_rope_ln_bwd on copies of the inputs placed `offset` bf16 elements into their buffers: offset 2 (4 bytes)
    keeps the generic kernel's bf16x2 accesses aligned but breaks the 16-byte alignment the vectorised kernel needs."""
    rows, C = x.shape

    def place(t):
        b = torch.empty(t.numel() + offset, dtype=BF16, device=DEV)
        b[offset:].copy_(t.flatten())
        return b[offset:].view(t.shape)
    xs, g0s, g1s, g2s, adds = (place(t) for t in (x, g0, g1, g2, add))
    dx = Guarded((rows, C), BF16, 64 * C, offset=offset)
    dg, db = Guarded((C,), F32T, 64 * C, dg0), Guarded((C,), F32T, 64 * C, db0)
    _call('og_rope_ln_bwd', xs.data_ptr(), freq.data_ptr(), gamma.data_ptr(), 1e-5, g0s.data_ptr(), g1s.data_ptr(),
          g2s.data_ptr(), adds.data_ptr(), dx.ptr(), dg.ptr(), db.ptr(), rows, C, pos_div, pos_mod, None)
    torch.cuda.synchronize()
    for n, o in (('dx', dx), ('dgamma', dg), ('dbeta', db)):
        o.check_guard(n)
    return {'dx': dx.t, 'dgamma': dg.t, 'dbeta': db.t}


@GPU
@pytest.mark.parametrize('mode', ['1d', '2d'])
@pytest.mark.parametrize('C', [128, 256, 512])
def test_rope_ln_bwd_all_gradient_inputs(C, mode):
    """g0, g1, g2 and add all given (the product always passes them), 105 rows (not a multiple of 8 warps), dgamma /
    dbeta pre-filled; aligned (vectorised kernel for C in {256, 512}) and misaligned (generic kernel) runs."""
    B, T, H, W = 1, 5, 7, 3
    rows = B * T * H * W
    pos_div, pos_mod = (H * W, T) if mode == '1d' else (1, H * W)
    x, g0, g1, g2, add = (_rand((rows, C), 10000 + C + i) for i in range(5))
    freq = O.rope_freq(C, mode).to(DEV)
    gamma, beta = _rope_ln_inputs(C, 10100 + C)
    dg0, db0 = _rand((C,), 10200 + C).float(), _rand((C,), 10300 + C).float()
    pos = (torch.arange(rows, device=DEV) // pos_div) % pos_mod
    st = rope_ln_ref(x.double(), pos, freq, gamma, beta)
    g = g0.double() + g1.double() + g2.double()
    ex = rope_ln_bwd_expect(st, g, gamma, add.double(), dg_init=dg0, db_init=db0)
    for offset in (0, 2):
        check_all(_rope_ln_bwd_call(x, freq, gamma, g0, g1, g2, add, dg0, db0, pos_div, pos_mod, offset), ex)


# ------------------------------------------------------------------------------------------------------------------
# composed autograd functions (ops.py) against a float64 emulation with the product's bf16 rounding points
# ------------------------------------------------------------------------------------------------------------------
def _composed_backward_expect(st, dy, gamma, grads, errs):
    """The product rounds dq, dk, dv to bf16 and feeds them with `add` = dy into og_rope_ln_bwd. Each intermediate is
    within (its kernel bound + U |value|) of the float64 value; that bound goes through |d dx / d g|."""
    g = sum(grads)
    eg = sum(e + U * t.abs() for t, e in zip(grads, errs))
    return rope_ln_bwd_expect(st, g, gamma, dy.double().reshape(g.shape), eg=SLACK * eg)


@GPU
@pytest.mark.parametrize('cond', [False, True])
def test_time_attention_res_composed(cond):
    from open_genie_b200 import ops
    B, T, H, W, nh, d = 2, 16, 8, 8, 4, 64
    C, P, scale = nh * d, H * W, nh * d ** -0.5
    x = _rand((B, T, H, W, C), 11000).requires_grad_(True)
    freq = O.rope_freq(C, '1d').to(DEV)
    gamma, beta = (t.requires_grad_(True) for t in _rope_ln_inputs(C, 11001))
    kc = vc = None
    if cond:
        kc = _rand((B, T, C), 11002).float().requires_grad_(True)
        vc = _rand((B, T, C), 11003).float().requires_grad_(True)
    y = ops.time_attention_res(x, freq, gamma, beta, nh, scale, kc, vc)
    q = y.grad_fn.saved_tensors[1]          # the bf16 LayerNorm(RoPE(x)) the product attends with
    dy = _rand(y.shape, 11004)
    y.backward(dy)
    torch.cuda.synchronize()
    rows = B * T * P
    pos = (torch.arange(rows, device=DEV) // P) % T
    st = rope_ln_ref(x.detach().double().reshape(rows, C), pos, freq, gamma.detach(), beta.detach())
    q_tol = bf16_tol(F_LN * (gamma.detach().double().abs() * (st['xh'].abs() + 1) + beta.detach().double().abs()),
                     st['y'])
    check('q', q.reshape(rows, C), st['y'], q_tol)
    q4, x4, dy4 = q.view(B, T, P, C), x.detach().view(B, T, P, C), dy.view(B, T, P, C)
    k4, v4 = (kc.detach().to(BF16), vc.detach().to(BF16)) if cond else (q4, q4)
    ex = temporal_expect(q4, k4, v4, dy4, x4, nh, scale, bcast=cond)
    check('y', y.detach().view(B, T, P, C), *ex['out_res'])
    names = ('dq',) if cond else ('dq', 'dk', 'dv')
    grads = [ex[n][0].reshape(rows, C) for n in names]
    errs = [(ex[n][1] / SLACK - U * ex[n][0].abs()).reshape(rows, C) for n in names]   # the pre-rounding bounds
    exb = _composed_backward_expect(st, dy, gamma.detach(), grads, errs)
    check_all({'dx': x.grad.reshape(rows, C), 'dgamma': gamma.grad, 'dbeta': beta.grad}, exb)
    if cond:
        check('dk_cond', kc.grad, *ex['dk_bcast'])
        check('dv_cond', vc.grad, *ex['dv_bcast'])


@GPU
def test_space_attention_res_composed():
    from open_genie_b200 import ops
    B, T, H, W, nh = 1, 2, 10, 10, 4
    C, S, scale = 64 * nh, H * W, nh * 64 ** -0.5
    x = _rand((B, T, H, W, C), 12000).requires_grad_(True)
    freq = O.rope_freq(C, '2d').to(DEV)
    gamma, beta = (t.requires_grad_(True) for t in _rope_ln_inputs(C, 12001))
    y = ops.space_attention_res(x, freq, gamma, beta, nh, scale)
    q = y.grad_fn.saved_tensors[1]
    dy = _rand(y.shape, 12002)
    y.backward(dy)
    torch.cuda.synchronize()
    rows, nseq = B * T * S, B * T
    pos = torch.arange(rows, device=DEV) % S
    st = rope_ln_ref(x.detach().double().reshape(rows, C), pos, freq, gamma.detach(), beta.detach())
    q_tol = bf16_tol(F_LN * (gamma.detach().double().abs() * (st['xh'].abs() + 1) + beta.detach().double().abs()),
                     st['y'])
    check('q', q.reshape(rows, C), st['y'], q_tol)
    q3, x3, dy3 = q.view(nseq, S, C), x.detach().view(nseq, S, C), dy.view(nseq, S, C)
    ex = flash_expect(q3, q3, q3, dy3, x3, nh, scale)
    check('y', y.detach().view(nseq, S, C), *ex['out_res'])
    grads = [ex[n][0].reshape(rows, C) for n in ('dq', 'dk', 'dv')]
    errs = [(ex[n][1] / SLACK - U * ex[n][0].abs()).reshape(rows, C) for n in ('dq', 'dk', 'dv')]
    exb = _composed_backward_expect(st, dy, gamma.detach(), grads, errs)
    check_all({'dx': x.grad.reshape(rows, C), 'dgamma': gamma.grad, 'dbeta': beta.grad}, exb)


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran: one profiled call per dispatch class
# ------------------------------------------------------------------------------------------------------------------
def _kernels_run(fn):
    """Names of the kernels two calls of `fn` launch. Late in a long test process the trace of a session sometimes
    lacked the kernels of its first call (the library's launch counter showed that they had run); those of a second,
    identical call were listed."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


def _temporal_once(d, T):
    return lambda: temporal_run(B=1, T=T, P=5, nh=2, d=d, bcast=0, seed=13000 + d + T)


def _rope_once(C, offset):
    def run():
        rows = 24
        x, g0, g1, g2, add = (_rand((rows, C), 13100 + i) for i in range(5))
        gamma, _ = _rope_ln_inputs(C, 13105)
        z = torch.zeros(C, device=DEV)
        _rope_ln_bwd_call(x, O.rope_freq(C, '1d').to(DEV), gamma, g0, g1, g2, add, z, z, 1, rows, offset)
    return run


PINS = {
    # class: (run, kernel names that must appear, names that must not)
    'temporal_mma': (_temporal_once(64, 16), ['og_temporal_attn_fwd_mma_kernel', 'og_temporal_attn_bwd_mma_kernel'],
                     ['og_temporal_attn_fwd_kernel<', 'og_temporal_attn_bwd_kernel<']),
    'temporal_lane64': (_temporal_once(64, 17), ['og_temporal_attn_fwd_kernel<64>', 'og_temporal_attn_bwd_kernel<64>'],
                        ['_mma_kernel']),
    'temporal_lane32': (_temporal_once(32, 16), ['og_temporal_attn_fwd_kernel<32>', 'og_temporal_attn_bwd_kernel<32>'],
                        ['_mma_kernel']),
    'flash': (lambda: flash_run(nseq=1, S=65, nh=1, seed=13200),
              ['og_flash_attn_fwd_kernel', 'og_flash_attn_bwd_kernel<0>', 'og_flash_attn_bwd_kernel<1>'], []),
    'rope_ln_bwd_vec': (_rope_once(512, 0), ['og_rope_ln_bwd_vec_kernel<2>'], []),
    'rope_ln_bwd_generic': (_rope_once(512, 2), ['og_rope_ln_bwd_kernel('], ['og_rope_ln_bwd_vec_kernel']),
}


@GPU
@pytest.mark.parametrize('cls', sorted(PINS))
def test_dispatch_kernel_names(cls):
    """The shapes the tests above use for each path still reach that path's kernel."""
    run, want, absent = PINS[cls]
    names = _kernels_run(run)
    for w in want:
        assert any(w in n for n in names), (cls, w, sorted(set(n for n in names if 'og_' in n)))
    for a in absent:
        assert not any(a in n for n in names), (cls, a, sorted(set(n for n in names if 'og_' in n)))
