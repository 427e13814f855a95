"""The LFQ quantiser and its entropy + commitment loss (csrc/lfq.cu) against an explicit float64 reference, element by
element.

Paths covered: og_lfq_fwd in inference (sign output, no workspace) and in training (straight-through output, loss,
workspace), the fp32 and bf16 outputs with a padded bf16 pitch, og_lfq_bwd with fp32 and bf16 dx (padded pitch,
zeroed pad columns), with and without gloss and dout; every codebook size D = 1..20 (odd D: a rectangular batch-mean
GEMM, H = 2^ceil(D/2) != L; D = 1: L = 1; D = 19, 20: 1024-entry halves), token counts that are not a multiple of the
SGEMM's 64 x 64 tiles, ntok = 1, ldx > D; flat, intermediate (a few per cent of the probability mass below the clamp
eps, so that whole rows are skipped and the closed form -log(eps) * mass is used) and saturated (beta = 100 at unit
inputs) regimes; zeros and inputs large enough to overflow expf; and the autograd function of ops.py.

The reference restates LookupFreeQuantization.forward (reference quantization.py:77-133) in float64. At large D the
(tokens x 2^D) softmax is evaluated chunk by chunk as the exact outer product p[n] = a[n] (x) b[n] of the two halves'
sigmoid products, in two passes (the batch mean first, then each chunk's backward with dL/d avg fixed); gradients
come from float64 autograd. `test_chunked_reference_matches_literal_formula` pins it to the literal einsum + softmax.

Every tolerance is a per-element worst-case bound built from the rounding points of the kernels (`lfq_expect`). The
`test_tolerance_rejects_*` tests run on the CPU and show that each bound still rejects the mistakes it exists to catch.
"""
import ctypes
import math

import pytest
import torch

GPU = pytest.mark.gpu
DEV = 'cuda'
F32T, F64T, BF16 = torch.float32, torch.float64, torch.bfloat16

# Rounding model, as in test_gpu_attention_paths.py. F32 is one fp32 ulp (twice the unit roundoff), used per operation;
# a sequential fp32 sum of n terms is within gam(n) of the exact sum, relative to the sum of the terms' magnitudes.
# CUDA's expf is within 2 ulp and logf within 1 ulp (CUDA C Programming Guide, accuracy tables; no fast math here).
F32 = 2.0 ** -23
U = 2.0 ** -8           # bf16 unit roundoff
SLACK = 1.02            # second-order terms (an error that is itself rounded) are folded into this factor
# Absolute floor. A sigmoid factor whose expf overflows is exactly 0 in the kernel (1e-38 or less in the reference);
# the codes it multiplies carry less than 2^-100 of anything here.
TINY = 2.0 ** -100
EPS = 1e-6
LOG_EPS = math.log(EPS)
W = dict(wc=0.25, we=0.1, wd=1.0)       # the module's default loss weights


def gam(n):
    return n * F32



# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
def lfq_literal(x, beta, wc, we, wd):
    """quantization.py:93-131 literally on float64 x [N, D] (CPU, D <= 12): codebook einsum, softmax, entropies."""
    D = x.shape[1]
    bit_mask = 2 ** torch.arange(D - 1, -1, -1)
    codebook = 2 * ((torch.arange(2 ** D)[:, None] & bit_mask) != 0).to(x.dtype) - 1
    p = (2 * (x @ codebook.T) * beta).softmax(-1)
    ent = lambda q: -(q * q.clamp(min=EPS).log()).sum(-1)
    commit = ((x - x.sign().detach()) ** 2).mean()
    return (ent(p).mean() + wd * ent(p.mean(0))) * we + commit * wc


def _split(D, mut):
    """(D1, D2): the high half takes ceil(D/2) dimensions. Mutation 'split' gives it floor(D/2), dropping one."""
    return (D // 2 if 'split' in mut else (D + 1) // 2), D // 2


def _halves(x, beta, D1, D2):
    """a [N, 2^D1], b [N, 2^D2] (MSB first) and their per-entry relative error bounds ra, rb.
    sigmoid(+-t), t = 4 beta x: t is rounded once (|dt| <= F32/2 |t|, and d log sigmoid(t) / dt = 1 - sigmoid(t) =
    the other factor), expf adds 2 ulp, 1 + e and the division one rounding each: e_sp = sm |t| F32 + 4 F32."""
    t = 4 * beta * x
    sp, sm = torch.sigmoid(t), torch.sigmoid(-t)
    esp, esm = sm * t.abs() * F32 + 4 * F32, sp * t.abs() * F32 + 4 * F32

    def build(lo, n):
        v = torch.ones(x.shape[0], 1, dtype=x.dtype, device=x.device)
        r = torch.zeros_like(v)
        for i in range(lo, lo + n):
            v = torch.stack((v * sm[:, i, None], v * sp[:, i, None]), -1).flatten(1)
            r = torch.stack((r + esm[:, i, None], r + esp[:, i, None]), -1).flatten(1)
        return v, r
    (a, ra), (b, rb) = build(0, D1), build(D1, D2)
    return a, b, ra, rb


def _probs(x, beta, D1, D2):
    a, b, ra, rb = _halves(x, beta, D1, D2)
    p = (a[:, :, None] * b[:, None, :]).flatten(1)
    # products: D - 1 multiplications after the factors
    R = (ra[:, :, None] + rb[:, None, :]).flatten(1) + (D1 + D2) * F32
    skipped = (a * b.amax(1, keepdim=True) < EPS)[:, :, None].expand(-1, -1, b.shape[1]).flatten(1)
    return p, R, skipped


def _ent_rows(p, skipped, mut):
    """-sum_j p log max(p, eps) per token. Mutation 'skip_zero': skipped rows add 0 instead of -log(eps) * mass."""
    e = p * p.clamp(min=EPS).log()
    if 'skip_zero' in mut:
        e = torch.where(skipped, torch.zeros_like(e), e)
    return -e.sum(1)


def lfq_expect(x32, beta, wc, we, wd, gl=None, dout=None, mut=(), chunk_elems=1 << 24, with_dx=True):
    """Reference and worst-case bound of og_lfq_fwd / og_lfq_bwd (training) on these fp32 inputs [N, D].

    Returns {'loss': (ref, tol), 'dx': (ref [N, D], tol)} plus 'sub_eps' (the share of the probability mass below eps).
    gl: the loss gradient (None: 1); dout: fp32 [N, D] or None.
    `mut` names a deliberate mistake of the reference; only the sensitivity tests pass it:
      'split' (floor(D/2) dimensions in the high half), 'no_plus1' (d H(avg) / d avg without the +1 for avg >= eps),
      'skip_zero' (skipped rows add 0), '4beta' (twice the entropy gradient), 'commit_n' (MSE divided by N, not N D).

    Error model (per probability p_j of a token, relative error R_j from `_halves` and the D - 1 products):
      forward per-token entropy: pairs with p >= eps add p (log p - log eps) in one thread's sequential sum of up to
        H ceil(L / 128) terms, a 128-thread block sum and the closed form log(eps) (sum a)(sum b); each term is off by
        p (2 R_j + 4 F32) (|log p| + |log eps| + 1) and the sums by gam(k). A pair within its own error of eps may be
        classified either way; p log max(p, eps) is continuous there, so that costs nothing at first order.
      batch mean: an SGEMM entry is an N-term fma sum, off by sum_n p R / N + gam(N + 2) avg; H(avg) then by
        (avg error) (|log avg| + 1) and a 1024-thread sum.
      backward: m1 / w1 sum val_j = p (log p - log eps + 1) over p >= eps (relative error 2 R_j + 64 F32 plus the sum);
        here the classification matters: a pair within 2 R_j p of eps may add or drop val = eps. m2 / g2bar sum
        p_j G2_j through the U / V GEMMs (R_j + gam(H + L + 20)), with G2's own error from the batch mean and logf.
        tanh_d = sp - sm is off by sp e_sp + sm e_sm + F32. Where dimension d is saturated,
        dx_d = 2 beta (M_d - Gbar tanh_d) is a difference of two nearly equal terms, so the bound is relative to the
        terms' magnitudes, 2 beta (|M_d| + |Gbar| |tanh_d|), and never to |dx_d|.
      fp32 atomics add the per-token stats in any order: gam(N) of the sum of magnitudes, whatever the order.
    """
    dev = x32.device
    x = x32.double()
    N, D = x.shape
    D1, D2 = _split(D, mut)
    H, L = 2 ** D1, 2 ** D2
    nc = max(1, chunk_elems // (H * L))
    chunks = [slice(i, min(i + nc, N)) for i in range(0, N, nc)]
    q = x.sign()
    gl_v = 1.0 if gl is None else float(gl)
    k_sum = H * (-(-L // 128)) + H + L + 16          # the longest fp32 sum behind one token's entropy terms

    # pass 1: batch mean, per-token entropies and their bounds
    avg = torch.zeros(H * L, dtype=F64T, device=dev)
    avg_err = torch.zeros_like(avg)
    ent = torch.zeros(N, dtype=F64T, device=dev)
    ent_err = torch.zeros(N, dtype=F64T, device=dev)
    sub_eps = 0.0
    with torch.no_grad():
        for c in chunks:
            p, R, skipped = _probs(x[c], beta, D1, D2)
            avg += p.sum(0)
            avg_err += (p * R).sum(0)
            ent[c] = _ent_rows(p, skipped, mut)
            w = p.clamp(min=EPS).log().abs() + abs(LOG_EPS) + 1
            ent_err[c] = (p * (2 * R + 4 * F32 + gam(k_sum)) * w).sum(1)
            sub_eps += float(torch.where(p < EPS, p, torch.zeros_like(p)).sum())
    avg /= N
    avg_err = avg_err / N + gam(N + 2) * avg
    av = avg.clone().requires_grad_(True)
    h_avg = -(av * av.clamp(min=EPS).log()).sum()
    (g_avg,) = torch.autograd.grad(h_avg, av)
    lp = avg.clamp(min=EPS).log()
    if 'no_plus1' in mut:
        g_avg = -lp
    G2 = we * wd * g_avg.detach()                     # dL / d avg
    e_havg = (avg_err * (lp.abs() + 1)).sum() + gam(2 ** D // 1024 + 42) * (avg * (lp.abs() + 1)).sum()
    commit = ((x - q) ** 2).sum() / (N if 'commit_n' in mut else N * D)
    inp = ent.sum() / N
    loss = (inp + wd * h_avg.detach()) * we + commit * wc
    e_loss = (we * (ent_err.sum() + gam(N) * ent.abs().sum()) / N + we * wd * e_havg
              + wc * gam(N + 40) * commit
              + gam(8) * (abs(we * inp) + abs(we * wd * h_avg.detach()) + abs(wc * commit)))
    out = {'loss': (loss * gl_v, SLACK * abs(gl_v) * e_loss), 'sub_eps': sub_eps / N}
    if not with_dx:
        return out

    # pass 2: per chunk, d/dx of (per-token entropies) / N * we + p . G2 / N, with G2 fixed
    dx_ent = torch.zeros_like(x)
    gs = we * wd / N
    # relative error of log max(avg, eps) -> absolute error of G2 per code
    g2_err = gs * (avg_err / avg.clamp(min=EPS) + 2 * F32 * (lp.abs() + 1))
    we_n = we / N
    A = torch.zeros(N, dtype=F64T, device=dev)        # error of m1_d, m2_d (each d) and of w1, g2bar
    S1 = torch.zeros(N, dtype=F64T, device=dev)       # sum of val_j
    S2 = torch.zeros(N, dtype=F64T, device=dev)       # sum of p_j |G2_j|
    for c in chunks:
        xc = x[c].clone().requires_grad_(True)
        p, R, skipped = _probs(xc, beta, D1, D2)
        Lc = we_n * _ent_rows(p, skipped, mut).sum() + (p @ G2).sum() / N
        (g,) = torch.autograd.grad(Lc, xc)
        dx_ent[c] = g
        with torch.no_grad():
            p, R = p.detach(), R.detach()
            big = p >= EPS
            val = torch.where(big, p * (p.log() - LOG_EPS + 1), torch.zeros_like(p))
            nb = ((p - EPS).abs() <= 2 * R * p).sum(1)
            S1[c] = val.sum(1)
            S2[c] = (p * G2.abs()).sum(1)
            A[c] = (we_n * ((val * (2 * R + 64 * F32 + gam(k_sum))).sum(1) + EPS * nb)
                    + (p * G2.abs() * (R + gam(H + L + 20))).sum(1) + p @ g2_err)
    if '4beta' in mut:
        dx_ent = 2 * dx_ent
    dcommit = wc * 2 * (x - q) / (N if 'commit_n' in mut else N * D)
    dx = gl_v * (dx_ent + dcommit)
    if dout is not None:
        dx = dx + dout.double()
    t = 4 * beta * x
    sp, sm = torch.sigmoid(t), torch.sigmoid(-t)
    esp, esm = sm * t.abs() * F32 + 4 * F32, sp * t.abs() * F32 + 4 * F32
    tanh = sp - sm
    dt = sp * esp + sm * esm + F32
    red_mag = we_n * (abs(LOG_EPS) * tanh.abs() + S1[:, None]) + S2[:, None]
    gbar_mag = (we_n * (abs(LOG_EPS) + S1) + S2)[:, None]
    e = 2 * beta * (A[:, None] * (1 + tanh.abs()) + we_n * abs(LOG_EPS) * dt + gbar_mag * dt
                    + gam(8) * (red_mag + gbar_mag * tanh.abs()))
    e = abs(gl_v) * (e + gam(6) * dcommit.abs()) + F32 * dx.abs()
    out['dx'] = (dx, SLACK * e)
    return out


def check(name, got, ref, tol):
    got = got.double().to(ref.device)
    ref = torch.as_tensor(ref, dtype=F64T, device=got.device)
    tol = torch.as_tensor(tol, dtype=F64T, device=got.device)
    assert got.shape == ref.shape, f'{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
    tol = tol + TINY
    bad = ~(err <= tol)    # NaN (an element never written) is bad too
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        ratio = (err / tol).flatten().nan_to_num(float('inf')).max().item()
        raise AssertionError(
            f'{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound, worst err/tol {ratio:.3g}; first at '
            f'flat index {i} (of shape {tuple(ref.shape)}): got {got.flatten()[i].item():.8g}, '
            f'ref {ref.flatten()[i].item():.8g}, tol {tol.flatten()[i].item():.3g}')


def _rejects(name, got, ref, tol):
    with pytest.raises(AssertionError):
        check(name, got, ref, tol)


# ------------------------------------------------------------------------------------------------------------------
# inputs: three regimes of beta |x|
# ------------------------------------------------------------------------------------------------------------------
# flat: 4 beta |x| ~ 4e-3, every code near 2^-D > eps for D <= 19, no row skipped; intermediate: at D = 18 a few per
# cent of the mass lies below eps (pinned by test_intermediate_regime_puts_mass_below_eps); saturated: the product's
# beta = 100 at unit-scale encoder outputs.
REGIMES = {'flat': 1e-5, 'intermediate': 4e-3, 'saturated': 0.5}
BETA = 100.0


def make_x(N, D, regime, seed, ld=None, device='cpu', extremes=False):
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn((N, D), generator=g, dtype=F64T) * REGIMES[regime]
    if extremes:
        # exact zeros (sign 0, index bit 0) and |x| large enough that expf(4 beta |x|) overflows to inf
        x.view(-1)[::7] = 0.0
        x.view(-1)[3::11] = 3e3 * torch.sign(torch.randn(x.view(-1)[3::11].shape, generator=g))
    x = x.float()
    if ld is not None and ld > D:
        full = torch.full((N, ld), float('nan'), dtype=F32T)
        full[:, :D] = x
        return full.to(device)
    return x.to(device)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference itself
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D', [1, 2, 5, 8, 11, 12])
@pytest.mark.parametrize('regime', ['flat', 'intermediate', 'saturated'])
def test_chunked_reference_matches_literal_formula(D, regime):
    """The chunked outer-product reference against the literal einsum + softmax of quantization.py, odd D included, so
    that its bit order and its D1 / D2 split cannot both be wrong in the same way as the kernel."""
    N = 13
    x32 = make_x(N, D, regime, 100 + D)
    x = x32.double().requires_grad_(True)
    loss = lfq_literal(x, BETA, **W)
    (dx,) = torch.autograd.grad(loss, x)
    ex = lfq_expect(x32, BETA, **W, chunk_elems=3 * 2 ** D)       # several chunks of 3 tokens
    assert torch.allclose(ex['loss'][0], loss, rtol=1e-12, atol=1e-15)
    assert torch.allclose(ex['dx'][0], dx, rtol=1e-9, atol=1e-15 * float(dx.abs().max()) + 1e-300)


def test_intermediate_regime_puts_mass_below_eps():
    """At D = 18 the intermediate regime has >= 1 % of the probability mass in codes below eps (closed-form rows)."""
    ex = lfq_expect(make_x(8, 18, 'intermediate', 7), BETA, **W, with_dx=False)
    assert ex['sub_eps'] >= 0.01, ex['sub_eps']
    assert lfq_expect(make_x(8, 18, 'flat', 7), BETA, **W, with_dx=False)['sub_eps'] == 0.0


# ------------------------------------------------------------------------------------------------------------------
# CPU: each bound rejects the mistakes it exists for
# ------------------------------------------------------------------------------------------------------------------
def _exact(ex):
    """What a correct kernel could return: the reference rounded to fp32."""
    return {k: ex[k][0].float() for k in ('loss', 'dx') if k in ex}


def test_tolerance_rejects_wrong_split_for_odd_d():
    for D in (5, 9, 11):
        x = make_x(16, D, 'intermediate', 200 + D)
        ex = lfq_expect(x, BETA, **W)
        got = _exact(ex)
        check('loss', got['loss'], *ex['loss'])
        check('dx', got['dx'], *ex['dx'])
        bad = lfq_expect(x, BETA, **W, mut=('split',))
        _rejects('loss', bad['loss'][0].float(), *ex['loss'])
        _rejects('dx', bad['dx'][0].float(), *ex['dx'])


def skipped_rows_x(N, D, seed, r=4.0):
    """Inputs that put much of the mass into skipped rows: the high half's dimensions at sigmoid(+-t) = r / (1 + r) (a
    row with several unlikely bits falls below eps / max b), the low half near 0 (b flat, max b = 2^-D2)."""
    g = torch.Generator().manual_seed(seed)
    D1 = (D + 1) // 2
    x = torch.zeros(N, D, dtype=F64T)
    sign = torch.randint(0, 2, (N, D1), generator=g) * 2 - 1
    x[:, :D1] = sign * math.log(r) / (4 * BETA) * (1 + 0.1 * torch.rand(N, D1, generator=g, dtype=F64T))
    x[:, D1:] = torch.randn(N, D - D1, generator=g, dtype=F64T) * 1e-5
    return x.float()


def test_tolerance_rejects_missing_plus_one_in_batch_entropy_gradient():
    # the +1 only matters for codes whose batch mean is below eps while the tokens put mass on them: one token
    x = skipped_rows_x(1, 18, 300)
    ex = lfq_expect(x, BETA, **W)
    check('dx', _exact(ex)['dx'], *ex['dx'])
    bad = lfq_expect(x, BETA, **W, mut=('no_plus1',))
    _rejects('dx', bad['dx'][0].float(), *ex['dx'])


def test_tolerance_rejects_skipped_rows_adding_zero():
    x = skipped_rows_x(4, 16, 400)
    ex = lfq_expect(x, BETA, **W, with_dx=False)
    assert ex['sub_eps'] > 1e-3
    check('loss', _exact(ex)['loss'], *ex['loss'])
    bad = lfq_expect(x, BETA, **W, mut=('skip_zero',), with_dx=False)
    _rejects('loss', bad['loss'][0].float(), *ex['loss'])


@pytest.mark.parametrize('regime', ['flat', 'intermediate', 'saturated'])
def test_tolerance_rejects_four_beta_in_backward(regime):
    x = make_x(16, 10, regime, 500)
    ex = lfq_expect(x, BETA, **W)
    check('dx', _exact(ex)['dx'], *ex['dx'])
    bad = lfq_expect(x, BETA, **W, mut=('4beta',))
    _rejects('dx', bad['dx'][0].float(), *ex['dx'])


def test_tolerance_rejects_commitment_divided_by_n():
    x = make_x(16, 10, 'saturated', 600)
    ex = lfq_expect(x, BETA, **W)
    bad = lfq_expect(x, BETA, **W, mut=('commit_n',))
    _rejects('loss', bad['loss'][0].float(), *ex['loss'])
    _rejects('dx', bad['dx'][0].float(), *ex['dx'])


# ------------------------------------------------------------------------------------------------------------------
# CPU: host-side argument validation
# ------------------------------------------------------------------------------------------------------------------
def test_lfq_argument_validation_returns_status_codes():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error())
    for D in (0, 21):
        bad(lib.og_lfq_fwd(p, 32, 4, D, 100.0, 0, .25, .1, 1., p, None, 0, p, None, None, None), b'outside [1,20]')
        bad(lib.og_lfq_bwd(p, 32, 4, D, 100.0, .25, .1, None, None, 0, p, None, 32, p, None), b'outside [1,20]')
        assert lib.og_lfq_workspace_bytes(4, D) == 0
    # training without a workspace, or without a loss
    bad(lib.og_lfq_fwd(p, 18, 4, 18, 100.0, 1, .25, .1, 1., p, None, 0, p, p, None, None), b'training needs')
    bad(lib.og_lfq_fwd(p, 18, 4, 18, 100.0, 1, .25, .1, 1., p, None, 0, p, None, p, None), b'training needs')
    # ld_dx < D; no dx at all; no workspace; no tokens
    bad(lib.og_lfq_bwd(p, 18, 4, 18, 100.0, .25, .1, None, None, 0, p, None, 17, p, None), b'bad arguments')
    bad(lib.og_lfq_bwd(p, 18, 4, 18, 100.0, .25, .1, None, None, 0, None, None, 18, p, None), b'bad arguments')
    bad(lib.og_lfq_bwd(p, 18, 4, 18, 100.0, .25, .1, None, None, 0, p, None, 18, None, None), b'bad arguments')
    bad(lib.og_lfq_fwd(p, 18, 0, 18, 100.0, 0, .25, .1, 1., p, None, 0, p, None, None, None), b'bad arguments')
    assert lib.og_lfq_workspace_bytes(4, 1) > 0 and lib.og_lfq_workspace_bytes(4, 20) > 0


# ------------------------------------------------------------------------------------------------------------------
# GPU: the C ABI
# ------------------------------------------------------------------------------------------------------------------
def _stream():
    return torch.cuda.current_stream().cuda_stream


def lfq_run(x, D, training, gloss=None, dout=None, ld_bf16=0, out_f32=True, dx_f32=True, dx_bf16=False, ld_dx=None,
            backward=True):
    """og_lfq_fwd (+ og_lfq_bwd) on fp32 x [N, ldx] (first D columns). Every output starts as NaN."""
    from open_genie_b200 import _lib
    N, ldx = x.shape
    r = {}
    out = torch.full((N, D), float('nan'), dtype=F32T, device=DEV) if out_f32 else None
    ob = torch.full((N, ld_bf16), float('nan'), dtype=BF16, device=DEV) if ld_bf16 else None
    idx = torch.full((N,), -7, dtype=torch.int64, device=DEV)
    loss = torch.full((1,), float('nan'), dtype=F32T, device=DEV)
    ws = None
    if training:
        ws = torch.full((_lib.load().og_lfq_workspace_bytes(N, D) // 4,), float('nan'), dtype=F32T, device=DEV)
    ptr = lambda t: None if t is None else t.data_ptr()
    _lib.call('og_lfq_fwd', x.data_ptr(), ldx, N, D, BETA, int(training), W['wc'], W['we'], W['wd'], ptr(out), ptr(ob),
              ld_bf16, idx.data_ptr(), ptr(loss) if training else None, ptr(ws), _stream())
    r.update(idx=idx, out=out, out_bf16=ob)
    if training:
        r['loss'] = loss[0]
    if training and backward:
        ld_dx = ld_dx or D
        gl = None if gloss is None else torch.tensor([gloss], dtype=F32T, device=DEV)
        dxf = torch.full((N, ld_dx), float('nan'), dtype=F32T, device=DEV) if dx_f32 else None
        dxb = torch.full((N, ld_dx), float('nan'), dtype=BF16, device=DEV) if dx_bf16 else None
        ld_dout = 0 if dout is None else dout.shape[1]
        _lib.call('og_lfq_bwd', x.data_ptr(), ldx, N, D, BETA, W['wc'], W['we'], ptr(gl), ptr(dout), ld_dout,
                  ptr(dxf), ptr(dxb), ld_dx, ws.data_ptr(), _stream())
        r.update(dx=dxf, dx_bf16=dxb)
    torch.cuda.synchronize()
    return r


def _check_quantised(r, x, D, training):
    """Indices (MSB first) and the quantised output: bit exact."""
    xs = x[:, :D].cpu()
    bits = (xs > 0).long() * 2 ** torch.arange(D - 1, -1, -1)
    assert torch.equal(r['idx'].cpu(), bits.sum(1))
    q = xs.sign()
    code = xs + (q - xs) if training else q          # fp32, evaluated like the reference's STE
    if r['out'] is not None:
        assert torch.equal(r['out'].cpu(), code)
    if r['out_bf16'] is not None:
        ob = r['out_bf16'].cpu()
        assert torch.equal(ob[:, :D], code.to(BF16))
        assert bool((ob[:, D:].float() == 0).all())            # pad columns exactly zero (not NaN, not -0 left over)


def _check_training(r, x, D, gloss=None, dout=None, ld_dx=None):
    ex = lfq_expect(x[:, :D].contiguous(), BETA, **W, gl=gloss, dout=None if dout is None else dout[:, :D])
    check('loss', r['loss'] * (1.0 if gloss is None else gloss), *ex['loss'])
    ref, tol = ex['dx']
    if r.get('dx') is not None:
        check('dx', r['dx'][:, :D], ref, tol)
        assert bool((r['dx'][:, D:] == 0).all())
    if r.get('dx_bf16') is not None:
        check('dx_bf16', r['dx_bf16'][:, :D], ref, SLACK * (tol + U * ref.abs()))
        assert bool((r['dx_bf16'][:, D:].float() == 0).all())
    return ex


@GPU
@pytest.mark.parametrize('D', list(range(1, 21)))
def test_every_codebook_size(D):
    """D = 1..20 at 37 tokens (not a multiple of the SGEMM tile), in inference and training, intermediate regime."""
    x = make_x(37, D, 'intermediate', 1000 + D, device=DEV)
    _check_quantised(lfq_run(x, D, training=False), x, D, False)
    r = lfq_run(x, D, training=True)
    _check_quantised(r, x, D, True)
    _check_training(r, x, D)


@GPU
@pytest.mark.parametrize('regime', list(REGIMES))
@pytest.mark.parametrize('D', [7, 12, 18])
def test_regimes(D, regime):
    x = make_x(100, D, regime, 2000 + D, device=DEV)
    r = lfq_run(x, D, training=True)
    _check_quantised(r, x, D, True)
    _check_training(r, x, D)


# D = 17..20 at the product's token counts (512 = B 2, 2048 = the benchmark's B 8 on a 4x8x8 latent), 8192, and
# ragged counts. The float64 reference dominates the run time (about 8 s for D = 20 at 8192 tokens on an H100).
PRODUCT = [(D, n) for D in (17, 18, 19, 20) for n in (512, 2048, 2049, 8191, 8192)]


@GPU
@pytest.mark.parametrize('D,N', PRODUCT)
def test_product_token_counts(D, N):
    regime = 'saturated' if N % 2 == 0 else 'intermediate'
    x = make_x(N, D, regime, 3000 + D + N, device=DEV)
    r = lfq_run(x, D, training=True)
    _check_quantised(r, x, D, True)
    _check_training(r, x, D)


@GPU
@pytest.mark.parametrize('D', [1, 11, 18, 20])
def test_single_token(D):
    x = make_x(1, D, 'intermediate', 4000 + D, device=DEV)
    _check_quantised(lfq_run(x, D, training=False), x, D, False)
    r = lfq_run(x, D, training=True)
    _check_quantised(r, x, D, True)
    _check_training(r, x, D)


@GPU
@pytest.mark.parametrize('D', [5, 18])
def test_strided_input_and_padded_outputs(D):
    """ldx > D (NaN in the columns beyond D), the bf16 output with ld_bf16 > D, fp32 + bf16 dx with ld_dx > D, gloss
    set and dout with ld_dout > D."""
    N = 70
    x = make_x(N, D, 'intermediate', 5000 + D, ld=D + 3, device=DEV)
    _check_quantised(lfq_run(x, D, training=False, ld_bf16=D + 6), x, D, False)
    g = torch.Generator(device='cpu').manual_seed(5100 + D)
    dout = torch.randn((N, D + 5), generator=g).mul(1e-3).to(DEV)
    dout[:, D:] = float('nan')                       # columns the kernel must not read
    r = lfq_run(x, D, training=True, ld_bf16=D + 6, gloss=0.75, dout=dout, dx_bf16=True, ld_dx=D + 4)
    _check_quantised(r, x, D, True)
    _check_training(r, x, D, gloss=0.75, dout=dout)
    # bf16 dx alone, no fp32 dx, no gloss, no dout
    r = lfq_run(x, D, training=True, out_f32=False, ld_bf16=D, dx_f32=False, dx_bf16=True, ld_dx=D + 2)
    _check_quantised(r, x, D, True)
    _check_training(r, x, D)


@GPU
@pytest.mark.parametrize('D', [6, 18])
def test_zeros_and_overflowing_inputs(D):
    """Exact zeros and |x| = 3000 (expf(4 beta |x|) = inf): finite results within the bounds, no NaN."""
    x = make_x(64, D, 'intermediate', 6000 + D, device=DEV, extremes=True)
    _check_quantised(lfq_run(x, D, training=False), x, D, False)
    r = lfq_run(x, D, training=True)
    _check_quantised(r, x, D, True)
    assert bool(torch.isfinite(r['loss'])) and bool(torch.isfinite(r['dx']).all())
    _check_training(r, x, D)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the autograd function
# ------------------------------------------------------------------------------------------------------------------
@GPU
def test_ops_lfq_backward_without_loss_or_output():
    from open_genie_b200 import ops
    D, N = 18, 300
    x0 = make_x(N, D, 'intermediate', 7000, device=DEV)
    g = torch.Generator(device='cpu').manual_seed(7001)
    gq = torch.randn((N, D), generator=g).to(DEV)
    # only the quantised output is used: dx = the straight-through gradient, exactly
    x = x0.clone().requires_grad_(True)
    out, idx, loss = ops.lfq(x, D, BETA, True, W['wc'], W['we'], W['wd'])
    (out * gq).sum().backward()
    assert torch.equal(x.grad, gq)
    # only the loss is used: dx = dloss / dx
    x = x0.clone().requires_grad_(True)
    out, idx, loss = ops.lfq(x, D, BETA, True, W['wc'], W['we'], W['wd'])
    loss.backward()
    ex = lfq_expect(x0, BETA, **W)
    check('loss', loss, *ex['loss'])
    check('dx', x.grad, *ex['dx'])
    # both, through the module
    from open_genie_b200.module.quantization import LookupFreeQuantization
    m = LookupFreeQuantization(D, input_dim=D).to(DEV).train()
    x = x0.clone().requires_grad_(True)
    (q, idx), loss = m(x)
    (loss * 0.5 + (q * gq).sum()).backward()
    ex = lfq_expect(x0, BETA, **W, gl=0.5, dout=gq)
    check('module loss', loss * 0.5, *ex['loss'])
    check('module dx', x.grad, *ex['dx'])
    # eval: sign output, no loss, no gradient path
    m.eval()
    (q, idx), loss = m(x0)
    assert loss is None and torch.equal(q, x0.sign())


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
@GPU
def test_dispatch_kernel_names():
    """The training cases reach the forward, batch-mean entropy and backward kernels and the SGEMM (one launch for
    the batch mean, two for U and V)."""
    from test_gpu_attention_paths import _kernels_run
    from open_genie_b200 import _lib
    x = make_x(37, 11, 'intermediate', 8000, device=DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    names = _kernels_run(lambda: lfq_run(x, 11, training=True))
    assert _lib.launch_count() - n0 == 2 * 6              # per call: forward, SGEMM, average; SGEMM x 2, backward
    for w in ('og_lfq_fwd_kernel', 'og_lfq_avg_kernel', 'og_lfq_bwd_kernel', 'og_sgemm_kernel'):
        assert any(w in n for n in names), (w, sorted(set(n for n in names if 'og_' in n)))
