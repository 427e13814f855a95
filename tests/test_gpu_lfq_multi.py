"""Multi-codebook lookup-free quantisation (num_codebook = C > 1, genie/module/quantization.py:39-133).

- Entry points: og_lfq_multi_fwd / og_lfq_multi_bwd against a float64 restatement of quantization.py:116-131 that
  materialises the reference's C * 2^D softmax (oracle.lfq_multi_oracle.lfq), for C = 2..4 and D = 1, 2, 5, 9, 10,
  and against the factorised float64 form at C = 2, D = 18 and 20; N = 1, odd N, padded pitches, bf16 outputs, with
  and without gloss and dout, in `Guarded` buffers. Indices and the straight-through output are bit-exact, the loss is
  held to 1e-3 relative and dx to a per-element bound built like test_gpu_lfq_paths.lfq_expect's. At C = 1 the new
  entry points are bit-identical to og_lfq_fwd / og_lfq_bwd.
- CPU: the factorised reference against the literal one, the bounds against the plausible mistakes (clamping at eps
  instead of C eps, one batch mean over all rows, normalising by N instead of R = N C, the commitment divided by N D,
  dropping log C, swapped codebook slices), the inputs' share of probabilities in [eps, C eps), argument checks with
  status codes, construction, state_dict keys and the refusals of LatentAction and Genie.
- Module and model level: tests/golden/lfq_multi.pt (oracle/make_golden_lfq_multi.py, the unmodified reference):
  the module cases, the mini tokenizer at (d_codebook, n_codebook) = (3, 2) and (6, 2), a GraphedTrainStep replay and
  codes_from_indices.
"""
import ctypes
import math

import pytest
import torch

from helpers import Guarded, det_weights, rel_l2
from oracle import fixtures as fx
from oracle import genie_oracle as O
from oracle import lfq_multi_oracle as LM

GPU = pytest.mark.gpu
DEV = 'cuda'
F32T, F64T, BF16 = torch.float32, torch.float64, torch.bfloat16
GOLDEN = 'lfq_multi.pt'

F32 = 2.0 ** -23
U = 2.0 ** -8
SLACK = 1.02
TINY = 2.0 ** -100
EPS = 1e-6
BETA = 100.0
W = dict(wc=0.25, we=0.1, wd=1.0)
LOSS_RTOL = 1e-3


def gam(n):
    return n * F32


# ------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------
def literal_loss(x, D, C, wc, we, wd):
    """quantization.py:116-131 on float64 x [N, C*D]: the C * 2^D softmax, materialised."""
    _, loss = LM.lfq(x[None], D, C, True, beta=BETA, commit_weight=wc, entropy_weight=we, diversity_weight=wd)
    return loss


def factorised_loss(x, D, C, wc, we, wd, mut=()):
    """The same loss in closed form on float64 x [N, C*D]. `mut` names a deliberate mistake (sensitivity tests only):
    'eps' (clamp at eps, not C eps), 'pooled' (one batch mean over all N C rows), 'norm_n' (per-row entropies summed
    and divided by N), 'commit_nd' (commitment divided by N D), 'no_logc' (no log C)."""
    N = x.shape[0]
    rows = x.reshape(N * C, D)
    q = LM.row_probs(rows, BETA)
    e = EPS if 'eps' in mut else C * EPS
    ent = lambda p: -(p * p.clamp(min=e).log()).sum(-1)
    h_rows = ent(q).sum() / (N if 'norm_n' in mut else N * C)
    h_avg = ent(q.mean(0)) if 'pooled' in mut else ent(q.reshape(N, C, -1).mean(0)).mean()
    logc = 0.0 if 'no_logc' in mut else math.log(C)
    commit = ((rows - rows.sign()) ** 2).sum() / (N * D if 'commit_nd' in mut else N * C * D)
    return we * (h_rows + wd * h_avg + (1 + wd) * logc) + wc * commit


def expect(x32, D, C, gl=None, dout=None, mut=(), literal=None):
    """Reference loss and dx of og_lfq_multi_fwd / og_lfq_multi_bwd (training) on fp32 x [N, C*D], with bounds.

    The loss is held to LOSS_RTOL relative. The dx bound follows test_gpu_lfq_paths.lfq_expect: every fp32 rounding
    of the kernels is bounded relative to the magnitude of the terms it enters, never relative to |dx| (dx of a
    saturated dimension is a difference of two nearly equal terms):
      rel = 2 R_j + 64 F32 + gam(longest sum), R_j <= D (4 F32 + max_t |t| sigmoid(-|t|) F32) the factor error;
      per row r and dimension d, with G2 = dL/d avg_c and q the row's distribution,
        S1 = sum_{q_j >= C eps} q_j (log q_j - log(C eps) + 1),  S2 = sum_j q_j |G2_j|,
        err_d = 2 beta gl [rel ((we/R)(|log C eps| (1 + |tanh_d|) + 2 S1) + 2 S2) + (we/R) C eps nb]
      where nb counts the codes within rel q of the clamp (classified either way). Plus rel |dcommit| + F32 |dx|.
    `literal`: take the reference through the materialised softmax (default for D <= 10), else the factorised form.
    `mut`: a mistake of factorised_loss, or 'swap' (dx of codebook slice c written to slice C - 1 - c)."""
    dev = x32.device
    x = x32.double()
    N = x.shape[0]
    R = N * C
    gl_v = 1.0 if gl is None else float(gl)
    xg = x.clone().requires_grad_(True)
    use_lit = literal if literal is not None else D <= 10
    if use_lit and not mut:
        loss = literal_loss(xg, D, C, W['wc'], W['we'], W['wd'])
    else:
        loss = factorised_loss(xg, D, C, W['wc'], W['we'], W['wd'], mut)
    (dx,) = torch.autograd.grad(loss, xg)
    loss = loss.detach()
    if 'swap' in mut:
        dx = dx.reshape(N, C, D).flip(1).reshape(N, C * D)
    dx = gl_v * dx
    if dout is not None:
        dx = dx + dout.double()
    out = {'loss': (gl_v * loss, LOSS_RTOL * abs(gl_v * float(loss)))}
    # magnitudes for the dx bound, from the factorised form
    with torch.no_grad():
        rows = x.reshape(R, D)
        q = LM.row_probs(rows, BETA)
        e = C * EPS
        avg = q.reshape(N, C, -1).mean(0)
        G2 = W['we'] * W['wd'] / R * (avg.clamp(min=e).log().abs() + 1)           # |dL/d avg_c|, [C, 2^D]
        t = 4 * BETA * rows
        tanh = torch.tanh(t / 2)
        H, L = 2 ** ((D + 1) // 2), 2 ** (D // 2)
        k_sum = H * (-(-L // 128)) + H + L + 16
        fac = D * (4 + float((t.abs() * torch.sigmoid(-t.abs())).max())) * F32
        rel = 2 * fac + 64 * F32 + gam(k_sum) + gam(H + L + 20) + gam(N + 2)
        big = q >= e
        S1 = torch.where(big, q * (q.log() - math.log(e) + 1), torch.zeros_like(q)).sum(1)
        S2 = (q.reshape(N, C, -1) * G2[None]).sum(-1).reshape(R)
        nb = ((q - e).abs() <= 2 * rel * q).sum(1).double()
        we_r = W['we'] / R
        mag = (we_r * (abs(math.log(e)) * (1 + tanh.abs()) + 2 * S1[:, None]) + 2 * S2[:, None])
        err = 2 * BETA * abs(gl_v) * (rel * mag + we_r * e * nb[:, None])
        dcommit = W['wc'] * 2 * (rows - rows.sign()) / (R * D)
        err = err + abs(gl_v) * (rel + gam(6)) * dcommit.abs()
        err = err.reshape(N, C * D) + F32 * dx.abs()
        band = float(((q >= EPS) & (q < e)).sum())
    out['dx'] = (dx, SLACK * err)
    out['band'] = band
    return out


def check(name, got, ref, tol):
    got = got.double().to(ref.device)
    tol = torch.as_tensor(tol, dtype=F64T, device=got.device)
    assert got.shape == ref.shape, f'{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
    tol = tol + TINY
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        ratio = (err / tol).flatten().nan_to_num(float('inf')).max().item()
        raise AssertionError(
            f'{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound, worst err/tol {ratio:.3g}; first at '
            f'flat index {i}: got {got.flatten()[i].item():.8g}, ref {ref.flatten()[i].item():.8g}, '
            f'tol {tol.flatten()[i].item():.3g}')


def _rejects(name, got, ref, tol):
    with pytest.raises(AssertionError):
        check(name, got, ref, tol)


# intermediate: 4 beta |x| ~ 1.6, so that codes spread from near 1 to far below the clamp
REGIMES = {'flat': 1e-5, 'intermediate': 4e-3, 'saturated': 0.5}


def make_x(N, D, C, regime, seed, ld=None, device='cpu'):
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = (torch.randn((N, C * D), generator=g, dtype=F64T) * REGIMES[regime]).float()
    if ld is not None and ld > C * D:
        full = torch.full((N, ld), float('nan'), dtype=F32T)
        full[:, :C * D] = x
        return full.to(device)
    return x.to(device)


def band_x(N, D, C, seed):
    """Inputs whose rows put many codes in [eps, C eps): every dimension at |4 beta x| = s with sigmoid(s) chosen so
    that the codes with half their bits unlikely sit at 1.5 eps."""
    g = torch.Generator().manual_seed(seed)
    k = D // 2
    # p_k = sigmoid(s)^(D-k) sigmoid(-s)^k = 1.5e-6 -> solve for s by bisection
    lo, hi = 0.0, 40.0
    for _ in range(200):
        s = (lo + hi) / 2
        lp = (D - k) * math.log(torch.sigmoid(torch.tensor(s, dtype=F64T)).item()) + \
            k * math.log(torch.sigmoid(torch.tensor(-s, dtype=F64T)).item())
        lo, hi = (s, hi) if lp > math.log(1.5e-6) else (lo, s)
    sign = torch.randint(0, 2, (N, C * D), generator=g, dtype=F64T) * 2 - 1
    jitter = 1 + 0.01 * torch.rand((N, C * D), generator=g, dtype=F64T)
    return (sign * s / (4 * BETA) * jitter).float()


# ------------------------------------------------------------------------------------------------------------------
# CPU: the references and their bounds
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D,C', [(1, 2), (2, 4), (5, 3), (9, 2), (10, 3)])
@pytest.mark.parametrize('regime', ['flat', 'intermediate', 'saturated'])
def test_factorised_reference_matches_literal_softmax(D, C, regime):
    x = make_x(7, D, C, regime, 100 + 10 * D + C).double().requires_grad_(True)
    lit = literal_loss(x, D, C, W['wc'], W['we'], W['wd'])
    (dl,) = torch.autograd.grad(lit, x)
    xf = x.detach().clone().requires_grad_(True)
    fac = factorised_loss(xf, D, C, W['wc'], W['we'], W['wd'])
    (df,) = torch.autograd.grad(fac, xf)
    assert torch.allclose(fac, lit, rtol=1e-12, atol=1e-15)
    assert torch.allclose(df, dl, rtol=1e-9, atol=1e-14 * float(dl.abs().max()) + 1e-300)


def test_inputs_hold_probabilities_between_eps_and_c_eps():
    """The intermediate regime and the band inputs put codes in [eps, C eps), where the clamp of C codebooks differs
    from the single-codebook one."""
    for D, C in ((9, 2), (10, 3), (10, 4)):
        assert expect(make_x(37, D, C, 'intermediate', 1000 + 10 * D + C), D, C)['band'] > 0, (D, C)
    assert expect(band_x(6, 10, 4, 7), 10, 4)['band'] > 6 * 4 * 100


def _exact(ex):
    return {k: ex[k][0].float() for k in ('loss', 'dx')}


@pytest.mark.parametrize('mut,D,C,regime', [
    ('pooled', 5, 3, 'intermediate'), ('norm_n', 9, 2, 'intermediate'), ('commit_nd', 5, 2, 'saturated'),
    ('no_logc', 2, 4, 'intermediate'), ('swap', 9, 2, 'intermediate')])
def test_bounds_reject_mistakes(mut, D, C, regime):
    x = make_x(37, D, C, regime, 600 + 10 * D + C)
    ex = expect(x, D, C)
    got = _exact(ex)
    check('loss', got['loss'], *ex['loss'])
    check('dx', got['dx'], *ex['dx'])
    bad = expect(x, D, C, mut=(mut,))
    if mut == 'no_logc':       # a constant: the loss moves, dx does not
        _rejects('loss', bad['loss'][0].float(), *ex['loss'])
    elif mut == 'swap':        # a permutation of the codebooks: dx moves, the loss does not
        _rejects('dx', bad['dx'][0].float(), *ex['dx'])
    else:
        _rejects('loss', bad['loss'][0].float(), *ex['loss'])
        _rejects('dx', bad['dx'][0].float(), *ex['dx'])


def test_bounds_reject_clamp_at_eps():
    """A flat row of 2^18 codes at 2^-18 = 3.8e-6 lies wholly inside [eps, 4 eps): the clamp at eps moves the loss by
    about 3e-3 relative (test_large_codebooks runs the kernels there). Where only a few codes fall in the band, the
    difference is below the fp32 rounding of the sums and no bound can see it."""
    x = make_x(3, 18, 4, 'flat', 9)
    ex = expect(x, 18, 4)
    check('loss', _exact(ex)['loss'], *ex['loss'])
    _rejects('loss', expect(x, 18, 4, mut=('eps',))['loss'][0].float(), *ex['loss'])


def test_swapped_slices_change_the_indices():
    x = make_x(37, 9, 2, 'intermediate', 11)
    bits = lambda t: ((t.reshape(37, 2, 9) > 0).long() * 2 ** torch.arange(8, -1, -1)).sum(-1)
    assert not torch.equal(bits(x), bits(x.reshape(37, 2, 9).flip(1).reshape(37, 18)))


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument checks
# ------------------------------------------------------------------------------------------------------------------
def test_multi_entry_points_reject_bad_arguments_with_status_codes():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error())
    fwd = lambda ldx, ntok, D, C, training=0, ob=None, ldb=0, loss=None, ws=None, x=p, idx=p: lib.og_lfq_multi_fwd(
        x, ldx, ntok, D, C, 100.0, training, .25, .1, 1., p, ob, ldb, idx, loss, ws, None)
    bwd = lambda ldx, ntok, D, C, dout=None, ldo=0, dxf=p, ldd=None, ws=p, x=p: lib.og_lfq_multi_bwd(
        x, ldx, ntok, D, C, 100.0, .25, .1, None, dout, ldo, dxf, None, C * D if ldd is None else ldd, ws, None)
    for D in (0, 21):
        bad(fwd(64, 4, D, 2), b'outside [1,20]')
        bad(bwd(64, 4, D, 2, ldd=64), b'outside [1,20]')
        assert lib.og_lfq_multi_workspace_bytes(4, D, 2) == 0
    for C in (0, -1, 65536):
        bad(fwd(64, 4, 4, C), b'n_codebook')
        bad(bwd(64, 4, 4, C, ldd=64), b'n_codebook')
        assert lib.og_lfq_multi_workspace_bytes(4, 4, C) == 0
    # no tokens; rows beyond an int
    bad(fwd(8, 0, 4, 2), b'ntok')
    bad(bwd(8, 0, 4, 2), b'ntok')
    bad(fwd(8, 2 ** 30, 4, 2), b'ntok')
    assert lib.og_lfq_multi_workspace_bytes(0, 4, 2) == 0 and lib.og_lfq_multi_workspace_bytes(2 ** 30, 4, 2) == 0
    # pitches below C * D
    bad(fwd(7, 4, 4, 2), b'ldx')
    bad(fwd(8, 4, 4, 2, ob=p, ldb=7), b'ld_bf16')
    bad(bwd(7, 4, 4, 2), b'ldx')
    bad(bwd(8, 4, 4, 2, ldd=7), b'ld_dx')
    bad(bwd(8, 4, 4, 2, dout=p, ldo=7), b'ld_dout')
    # training without a workspace or a loss; null pointers
    bad(fwd(8, 4, 4, 2, training=1, loss=p), b'training needs')
    bad(fwd(8, 4, 4, 2, training=1, ws=p), b'training needs')
    bad(fwd(8, 4, 4, 2, x=None), b'bad arguments')
    bad(fwd(8, 4, 4, 2, idx=None), b'bad arguments')
    bad(bwd(8, 4, 4, 2, ws=None), b'bad arguments')
    bad(bwd(8, 4, 4, 2, dxf=None), b'bad arguments')
    # sizes: size_t arithmetic, and C = 1 is the single-codebook workspace
    for ntok, D in ((4, 1), (37, 9), (2048, 18), (1 << 20, 20)):
        assert lib.og_lfq_multi_workspace_bytes(ntok, D, 1) == lib.og_lfq_workspace_bytes(ntok, D)
    H = L = 1 << 10
    assert lib.og_lfq_multi_workspace_bytes(1 << 20, 20, 2) == 4 * ((1 << 21) * (H + L) * 2 + (2 << 20) * 2 + 4)


# ------------------------------------------------------------------------------------------------------------------
# CPU: construction, keys, refusals
# ------------------------------------------------------------------------------------------------------------------
def test_module_keys_and_codebook_match_the_reference(golden):
    from open_genie_b200.module.quantization import LookupFreeQuantization
    g = golden(GOLDEN)
    for name, case in g['module'].items():
        m = LookupFreeQuantization(case['D'], num_codebook=case['C'], input_dim=case['input_dim'],
                                   use_bias=case['bias'])
        assert sorted(m.state_dict()) == case['keys'], name
        cb = m.codebook
        assert cb.shape == (case['C'] * 2 ** case['D'], case['D'])
        assert torch.equal(cb, cb[:2 ** case['D']].repeat(case['C'], 1))
    # the reference's default input_dim is C * 2^D: a projection
    m = LookupFreeQuantization(4, num_codebook=2)
    assert m.proj_inp.in_features == 32 and m.proj_inp.out_features == 8


def test_tokenizer_keys_match_the_reference(golden):
    import open_genie_b200 as og
    g = golden(GOLDEN)
    for name, case in g['tokenizer'].items():
        tok = og.VideoTokenizer(fx.MINI_ENC, fx.MINI_DEC, d_codebook=case['D'], n_codebook=case['C'],
                                gan_loss_weight=0, perc_loss_weight=0)
        assert sorted(tok.state_dict()) == case['keys'], name
        assert tok.quant.num_codebooks == case['C']


def test_latent_action_and_genie_refuse_several_codebooks():
    import open_genie_b200 as og
    from open_genie_b200.action import LatentAction
    with pytest.raises(NotImplementedError, match='LatentAction supports n_codebook = 1'):
        LatentAction(fx.MINI_ACT_ENC, fx.MINI_ACT_DEC, d_codebook=fx.MINI_ACT_D_CODEBOOK, n_embd=fx.MINI_ACT_EMBD,
                     inp_shape=fx.MINI_ACT_VIDEO_SHAPE[-2:], n_codebook=2)
    tok = og.VideoTokenizer(fx.MINI_ENC, fx.MINI_DEC, d_codebook=3, n_codebook=2, gan_loss_weight=0,
                            perc_loss_weight=0)
    with pytest.raises(NotImplementedError, match='n_codebook = 1'):
        og.Genie(tok, latent_action={}, dynamics_model={})


# ------------------------------------------------------------------------------------------------------------------
# GPU: the C ABI
# ------------------------------------------------------------------------------------------------------------------
def _stream():
    return torch.cuda.current_stream().cuda_stream


def multi_run(x, D, C, training, gloss=None, dout=None, ld_bf16=0, dx_bf16=False, ld_dx=None, single=False):
    """og_lfq_multi_fwd (+ og_lfq_multi_bwd) on fp32 x [N, ldx] into Guarded outputs; `single` calls og_lfq_fwd /
    og_lfq_bwd instead (C = 1)."""
    from open_genie_b200 import _lib
    N, ldx = x.shape
    lib = _lib.load()
    out = Guarded((N, C * D), F32T)
    ob = Guarded((N, ld_bf16), BF16) if ld_bf16 else None
    idx = Guarded((N, C), torch.float64)                   # int64 storage, NaN-patterned
    loss = Guarded((1,), F32T)
    ws = None
    if training:
        nb = lib.og_lfq_workspace_bytes(N, D) if single else lib.og_lfq_multi_workspace_bytes(N, D, C)
        ws = torch.full((nb // 4,), float('nan'), dtype=F32T, device=DEV)
    ptr = lambda t: None if t is None else t.ptr() if isinstance(t, Guarded) else t.data_ptr()
    head = (x.data_ptr(), ldx, N, D) if single else (x.data_ptr(), ldx, N, D, C)
    _lib.call('og_lfq_fwd' if single else 'og_lfq_multi_fwd', *head, BETA, int(training), W['wc'], W['we'], W['wd'],
              ptr(out), ptr(ob), ld_bf16, ptr(idx), ptr(loss) if training else None, ptr(ws), _stream())
    r = {'out': out, 'out_bf16': ob, 'idx': idx, 'loss': loss}
    if training:
        ld_dx = ld_dx or C * D
        gl = None if gloss is None else torch.tensor([gloss], dtype=F32T, device=DEV)
        dxf = Guarded((N, ld_dx), F32T)
        dxb = Guarded((N, ld_dx), BF16) if dx_bf16 else None
        ld_dout = 0 if dout is None else dout.shape[1]
        _lib.call('og_lfq_bwd' if single else 'og_lfq_multi_bwd', *head, BETA, W['wc'], W['we'], ptr(gl), ptr(dout),
                  ld_dout, ptr(dxf), ptr(dxb), ld_dx, ws.data_ptr(), _stream())
        r.update(dx=dxf, dx_bf16=dxb)
    torch.cuda.synchronize()
    for k, v in r.items():
        if isinstance(v, Guarded):
            v.check_guard(k)
    return r


def _check_quantised(r, x, D, C, training):
    N = x.shape[0]
    xs = x[:, :C * D].cpu()
    bits = ((xs.reshape(N, C, D) > 0).long() * 2 ** torch.arange(D - 1, -1, -1)).sum(-1)
    assert torch.equal(r['idx'].t.view(torch.int64).cpu(), bits)
    q = xs.sign()
    code = xs + (q - xs) if training else q
    assert torch.equal(r['out'].t.cpu(), code)
    if r['out_bf16'] is not None:
        ob = r['out_bf16'].t.cpu()
        assert torch.equal(ob[:, :C * D], code.to(BF16))
        assert bool((ob[:, C * D:].float() == 0).all())


def _check_training(r, x, D, C, gloss=None, dout=None, **kw):
    CD = C * D
    ex = expect(x[:, :CD].contiguous(), D, C, gl=gloss, dout=None if dout is None else dout[:, :CD], **kw)
    check('loss', r['loss'].t[0] * (1.0 if gloss is None else gloss), *ex['loss'])
    ref, tol = ex['dx']
    check('dx', r['dx'].t[:, :CD], ref, tol)
    assert bool((r['dx'].t[:, CD:] == 0).all())
    if r.get('dx_bf16') is not None:
        check('dx_bf16', r['dx_bf16'].t[:, :CD], ref, SLACK * (tol + U * ref.abs()))
        assert bool((r['dx_bf16'].t[:, CD:].float() == 0).all())
    return ex


@GPU
@pytest.mark.parametrize('C', [2, 3, 4])
@pytest.mark.parametrize('D', [1, 2, 5, 9, 10])
def test_codebooks_against_the_literal_softmax(D, C):
    """37 tokens (odd, not a multiple of the SGEMM tile), inference and training, intermediate regime."""
    x = make_x(37, D, C, 'intermediate', 2000 + 10 * D + C, device=DEV)
    _check_quantised(multi_run(x, D, C, training=False), x, D, C, False)
    r = multi_run(x, D, C, training=True)
    _check_quantised(r, x, D, C, True)
    _check_training(r, x, D, C)


@GPU
@pytest.mark.parametrize('regime', ['flat', 'saturated'])
@pytest.mark.parametrize('D,C', [(5, 3), (10, 2)])
def test_regimes(D, C, regime):
    x = make_x(64, D, C, regime, 2500 + 10 * D + C, device=DEV)
    r = multi_run(x, D, C, training=True)
    _check_quantised(r, x, D, C, True)
    _check_training(r, x, D, C)


@GPU
def test_probabilities_between_eps_and_c_eps():
    x = band_x(6, 10, 4, 7).to(DEV)
    r = multi_run(x, 10, 4, training=True)
    _check_quantised(r, x, 10, 4, True)
    _check_training(r, x, 10, 4)


@GPU
@pytest.mark.parametrize('D,C,N,regime', [(18, 2, 5, 'intermediate'), (20, 2, 3, 'intermediate'), (18, 4, 3, 'flat')])
def test_large_codebooks_against_the_factorised_form(D, C, N, regime):
    """C = 2 at D = 18 and 20; and D = 18, C = 4 with every code in [eps, 4 eps), where a clamp at eps is visible."""
    x = make_x(N, D, C, regime, 3000 + D + C, device=DEV)
    r = multi_run(x, D, C, training=True)
    _check_quantised(r, x, D, C, True)
    _check_training(r, x, D, C, literal=False)


@GPU
@pytest.mark.parametrize('D,C', [(1, 4), (5, 3), (10, 2)])
def test_single_token(D, C):
    x = make_x(1, D, C, 'intermediate', 4000 + 10 * D + C, device=DEV)
    _check_quantised(multi_run(x, D, C, training=False), x, D, C, False)
    r = multi_run(x, D, C, training=True)
    _check_quantised(r, x, D, C, True)
    _check_training(r, x, D, C)


@GPU
@pytest.mark.parametrize('D,C', [(5, 3), (9, 2)])
def test_padded_pitches_gloss_and_dout(D, C):
    """ldx > C D (NaN beyond), bf16 output with ld_bf16 > C D, fp32 + bf16 dx with ld_dx > C D, gloss and dout with
    ld_dout > C D; then the same without gloss and dout."""
    N, CD = 70, C * D
    x = make_x(N, D, C, 'intermediate', 5000 + 10 * D + C, ld=CD + 3, device=DEV)
    _check_quantised(multi_run(x, D, C, training=False, ld_bf16=CD + 6), x, D, C, False)
    g = torch.Generator(device='cpu').manual_seed(5100 + D)
    dout = torch.randn((N, CD + 5), generator=g).mul(1e-3).to(DEV)
    dout[:, CD:] = float('nan')
    r = multi_run(x, D, C, training=True, ld_bf16=CD + 6, gloss=0.75, dout=dout, dx_bf16=True, ld_dx=CD + 4)
    _check_quantised(r, x, D, C, True)
    _check_training(r, x, D, C, gloss=0.75, dout=dout)
    r = multi_run(x, D, C, training=True, ld_bf16=CD, dx_bf16=True, ld_dx=CD + 2)
    _check_quantised(r, x, D, C, True)
    _check_training(r, x, D, C)


@GPU
@pytest.mark.parametrize('D', [1, 5, 18, 20])
def test_one_codebook_is_bit_identical_to_the_single_entry_points(D):
    N = 53
    x = make_x(N, D, 1, 'intermediate', 6000 + D, ld=D + 2, device=DEV)
    g = torch.Generator(device='cpu').manual_seed(6100 + D)
    dout = torch.randn((N, D + 1), generator=g).mul(1e-3).to(DEV)
    kw = dict(gloss=0.5, dout=dout, ld_bf16=D + 3, dx_bf16=True, ld_dx=D + 2)
    a = multi_run(x, D, 1, training=True, single=True, **kw)
    b = multi_run(x, D, 1, training=True, **kw)
    for k in ('out', 'out_bf16', 'idx', 'dx', 'dx_bf16'):
        assert torch.equal(a[k].buf.view(torch.int8), b[k].buf.view(torch.int8)), k
    # the per-row entropy and commitment sums reach the loss through fp32 atomics, whose order varies from run to run
    # (og_lfq_fwd against itself too): the same terms, summed in another order
    la, lb = a['loss'].t[0].item(), b['loss'].t[0].item()
    assert abs(la - lb) <= 4 * N * F32 * abs(la), (la, lb)
    assert torch.equal(a['loss'].buf[1:].view(torch.int8), b['loss'].buf[1:].view(torch.int8))


@GPU
def test_launches_per_step():
    """Forward: rows, one batched SGEMM for all C batch means, entropy + loss; backward: two batched SGEMMs, rows."""
    from open_genie_b200 import _lib
    x = make_x(37, 5, 3, 'intermediate', 8000, device=DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    multi_run(x, 5, 3, training=True)
    assert _lib.launch_count() - n0 == 6


# ------------------------------------------------------------------------------------------------------------------
# GPU: module and model level against the reference's golden
# ------------------------------------------------------------------------------------------------------------------
@GPU
def test_module_cases_against_the_reference(golden):
    from open_genie_b200.module.quantization import LookupFreeQuantization
    g = golden(GOLDEN)
    for name, case in g['module'].items():
        D, C = case['D'], case['C']
        m = LookupFreeQuantization(D, num_codebook=C, input_dim=case['input_dim'], use_bias=case['bias'])
        det_weights(m)
        m.to(DEV)
        scale = 0.01 if case['input_dim'] == C * D else 1.0
        x0 = O.det_uniform(f'lfqm.x.{name}', case['shape'], scale)
        gout = O.det_uniform(f'lfqm.g.{name}', case['shape'], 1e-3).to(DEV)
        t = case['train']
        m.train()
        x = x0.to(DEV).requires_grad_(True)
        (out, idxs), loss = m(x, transpose=True)
        assert idxs.shape == t['idxs'].shape and idxs.dtype == torch.int64, name
        assert torch.equal(idxs.cpu(), t['idxs']), name
        assert torch.allclose(out.detach().cpu(), t['out'], rtol=1e-5, atol=1e-6), name
        assert abs(loss.item() - t['loss'].item()) <= LOSS_RTOL * abs(t['loss'].item()), (name, loss.item())
        (loss + (out * gout).sum()).backward()
        assert rel_l2(x.grad.cpu(), t['dx']) < 1e-3, (name, rel_l2(x.grad.cpu(), t['dx']))
        for k, p in m.named_parameters():
            assert rel_l2(p.grad.cpu(), t['grads'][k]) < 1e-3, (name, k)
        m.eval()
        (out, idxs), loss = m(x0.to(DEV), transpose=True)
        assert loss is None
        assert torch.equal(idxs.cpu(), case['eval']['idxs']), name
        assert torch.allclose(out.cpu(), case['eval']['out'], rtol=1e-5, atol=1e-6), name


def _mini(D, C):
    import open_genie_b200 as og
    tok = og.VideoTokenizer(fx.MINI_ENC, fx.MINI_DEC, d_codebook=D, n_codebook=C, gan_loss_weight=0,
                            perc_loss_weight=0)
    det_weights(tok)
    return tok.to(DEV)


@GPU
@pytest.mark.parametrize('D,C', [(3, 2), (6, 2)])
def test_mini_tokenizer_against_the_reference(golden, D, C):
    g = golden(GOLDEN)['tokenizer'][f'tok_d{D}c{C}']
    tok = _mini(D, C)
    video = O.det_uniform('tokenizer.video', fx.MINI_VIDEO_SHAPE).to(DEV)
    quant, idxs = tok.tokenize(video)
    assert tok.training
    assert quant.shape == g['quant'].shape and idxs.shape == g['idxs'].shape and idxs.dtype == torch.int64
    assert idxs.shape[-1] == C
    # a sign can only flip where the quantiser's input is below the accumulated bf16 conv error
    enc = g['enc'].movedim(1, -1)
    if 'quant.proj_inp.weight' in dict(tok.named_parameters()):
        sd = {k: v.cpu() for k, v in tok.state_dict().items()}
        enc = torch.nn.functional.linear(enc, sd['quant.proj_inp.weight'], sd['quant.proj_inp.bias'])
    enc = enc.unflatten(-1, (C, D))
    shifts = torch.arange(D - 1, -1, -1)
    bits = ((g['idxs'][..., None] >> shifts) & 1).bool()
    got = ((idxs.cpu()[..., None] >> shifts) & 1).bool()
    safe = enc.abs() > 0.05 * enc.abs().mean()
    assert torch.equal(bits[safe], got[safe]), 'sign flips on well-separated latents'
    assert (bits == got).float().mean().item() > 0.97
    # training loss and every gradient's norm (tolerances of test_gpu_tokenizer.py)
    loss, (rec, _, _, _, ql) = tok(video)
    loss.backward()
    assert abs(rec.item() - g['rec_loss'].item()) / g['rec_loss'].item() < 2e-2
    assert abs(ql.item() - g['quant_loss'].item()) / g['quant_loss'].item() < 5e-2
    assert abs(loss.item() - g['loss'].item()) / g['loss'].item() < 3e-2
    grads = {k: p.grad.float().cpu() for k, p in tok.named_parameters() if p.grad is not None}
    assert sorted(grads) == g['grad_names']
    for k, n in g['grad_norm'].items():
        if n <= 1e-6:
            continue
        r = grads[k].norm().item() / n
        # the decoder side (and proj_out) against the fp32 reference; the encoder side (and proj_inp) passes through
        # d/dx of the entropy at beta = 100, narrower than bf16 noise: scale only, as in test_gpu_tokenizer.py
        if k.startswith('dec_layers') or k.startswith('quant.proj_out'):
            assert abs(r - 1) < 0.05, (k, r)
        else:
            assert 0.5 < r < 2.0, (k, r)


@GPU
@pytest.mark.parametrize('D,C', [(3, 2), (6, 2)])
def test_codes_from_indices_equal_the_eval_quant(D, C):
    tok = _mini(D, C)
    video = O.det_uniform('tokenizer.video', fx.MINI_VIDEO_SHAPE).to(DEV)
    tok.eval()
    with torch.no_grad():
        (q, idxs), _ = tok.quant(tok.encode(video), transpose=True)
        codes = tok.quant.codes_from_indices(idxs)
    assert idxs.shape[-1] == C and codes.shape == q.shape
    assert torch.allclose(codes.float(), q.float(), rtol=1e-6, atol=1e-6)


@GPU
def test_graphed_train_step_replays_the_eager_step():
    from open_genie_b200 import ops
    from open_genie_b200.graph import GraphedTrainStep
    video = O.det_uniform('tokenizer.video', fx.MINI_VIDEO_SHAPE).to(DEV)
    try:
        tok = _mini(6, 2)
        step = GraphedTrainStep(tok, tok.configure_optimizers(), video, warmup=2)
        seen = []
        for _ in range(3):
            with torch.no_grad():
                expect_l = float(tok.training_step(video, 0))
            got = step(video).item()
            assert abs(got - expect_l) <= 5e-3 * abs(expect_l), (got, expect_l, seen)
            seen.append(got)
        assert len(set(seen)) == 3 and max(seen) - min(seen) > 1e-2 * abs(seen[0]), seen
    finally:
        ops.enable_zero_arena(False)
