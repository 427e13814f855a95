"""Every path of the GroupNorm / AdaGN / activation kernels (csrc/norm_act.cu) against an explicit float64 reference,
element by element.

Paths covered: the statistics kernels (one group per channel vector, and the per-channel kernel for (C/G) % 8 != 0),
the two-launch forms (og_gn_finalize + og_affine_act_fwd, og_gn_bwd_finalize + og_affine_act_bwd_apply) and the
one-launch forms (og_gn_act_fwd, og_gn_act_bwd) for the four activation codes, the backward reduction with every
workspace size (direct add, shrunk grid, full grid + og_sum_partials), the dx column sum, the pure activation
backward, the AdaGN conditioning kernels, and the autograd functions of ops.py.

Every tolerance is a per-element worst-case bound built from the rounding points of the path under test
(`gn_expect`, `adagn_expect`). The `test_tolerance(s)_reject_*` tests run on the CPU and show that each bound still
rejects the mistakes it exists to catch.
"""
import pytest
import torch
import torch.nn.functional as F

from helpers import Guarded

GPU = pytest.mark.gpu
DEV = 'cuda'
BF16, F32T, F64T = torch.bfloat16, torch.float32, torch.float64

# Rounding model, as in test_gpu_attention_paths.py. U is the unit roundoff of bf16 (8 significant bits). F32 is one
# fp32 ulp, used per operation (twice fp32's unit roundoff); a sequential fp32 sum of n terms is within gam(n) of the
# exact sum, relative to the sum of the terms' magnitudes.
U = 2.0 ** -8
F32 = 2.0 ** -23
# The fp64 combine of the statistics (shared and global atomics in any order): a few thousand additions at 2^-53 each.
# Far below every fp32 term; kept so that the bound does not claim more than the kernel does.
F64 = 2.0 ** -40
# tanh.approx.f32: the PTX ISA documents a maximum relative error of about 2^-11 (2^-10.987).
ETANH = 2.0 ** -10.98
SLACK = 1.02    # second-order terms (an error that is itself rounded, U * err) are folded into this factor
TINY = 2.0 ** -100
LEAKY = 0.01


def gam(n):
    return n * F32


# ------------------------------------------------------------------------------------------------------------------
# launch geometry: mirrors reduce_grid / partial_grid of norm_act.cu (kStatRows = 16)
# ------------------------------------------------------------------------------------------------------------------
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def reduce_grid(N, V, per_sm):
    """(blocks per sample, rows per block) of reduce_grid."""
    groups = -(-V // 16)
    want = min(max(-(-(per_sm * num_sms()) // N), 1), groups)
    gpb = -(-groups // want)
    return -(-groups // gpb), gpb * 16


def partial_grid(N, V, floats_per_block, ws_bytes):
    gx, rpb = reduce_grid(N, V, 6)
    fit = ws_bytes // 4 // floats_per_block if ws_bytes else 0
    if gx * N > fit:
        want = max(fit // N, 1)
        groups = -(-V // 16)
        gpb = -(-groups // want)
        gx, rpb = -(-groups // gpb), gpb * 16
    return gx, rpb


def layout(N, V, C, ws_reduce=None, ws_bwd=None, colsum=False):
    """Sum lengths and launch counts of one forward + backward chain.
    Ls: fp32 terms per thread of a statistics sum (8 channels x rows per thread).
    Lr: terms of an S entry: the rows of one thread, the row lanes of its block, then the blocks (og_sum_partials) or
        the add into S. Lc: the same for dx_colsum (its partials are one per block over all N samples)."""
    lanes = 256 // (C // 8)
    gs, rs = reduce_grid(N, V, 6)
    gr, rr = partial_grid(N, V, 2 * C, ws_reduce)
    if colsum:
        gb, rb = partial_grid(N, V, C, ws_bwd)
    else:
        gb, rb = reduce_grid(N, V, 6)
    rpt = lambda rpb: -(-min(rpb, V) // lanes)
    return {'Ls': 8 * rpt(rs) + 2, 'Lr': rpt(rr) + lanes + gr + 2, 'Lc': rpt(rb) + lanes + gb * N + 2,
            'reduce_partials': gr > 1, 'bwd_partials': colsum and gb * N > 1, 'gr': gr, 'gb': gb}


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
def act_fwd(pre, act, slope=LEAKY, silu_as_sigmoid=False):
    if act == 1:
        return torch.sigmoid(pre) if silu_as_sigmoid else pre * torch.sigmoid(pre)
    if act == 2:
        return torch.where(pre > 0, pre, slope * pre)
    if act == 3:
        return pre.clamp_min(0)
    return pre


def act_grad(pre, act, slope=LEAKY):
    if act == 1:
        s = torch.sigmoid(pre)
        return s * (1 + pre * (1 - s))
    if act == 2:
        return torch.where(pre > 0, torch.ones_like(pre), torch.full_like(pre, slope))
    if act == 3:
        return (pre > 0).to(pre.dtype)
    return torch.ones_like(pre)


def gn_ref(x, G, eps, act, gamma=None, beta=None, cs=None, csh=None, dy=None, add=None, mut=()):
    """Explicit GroupNorm(G) + AdaGN modulation + activation on x [N, V, C] (float64), and its backward for dy in
    closed form. gamma, beta: [C] or None; cs, csh: [N, C] or None; add: [N, V, C] or None.
    `mut` names a deliberate mistake; only the sensitivity tests pass it."""
    N, V, C = x.shape
    cpg = C // G
    ch = torch.arange(C, device=x.device)
    grp = ((ch + 1) // cpg).clamp(max=G - 1) if 'group_shift' in mut else ch // cpg
    oh = F.one_hot(grp, G).to(x.dtype)                   # [C, G]
    gs = lambda t: t @ oh                                 # per-(n, c) -> per-(n, g) sum over the group's channels
    bc = lambda t: t @ oh.T                               # per-(n, g) -> per-(n, c)
    cnt = V * oh.sum(0)                                   # [G] elements per group
    mean = gs(x.sum(1)) / cnt
    d = x - bc(mean)[:, None]
    var = gs((d * d).sum(1)) / (cnt - 1 if 'unbiased' in mut else cnt)
    rstd = var.rsqrt() + eps if 'eps_outside' in mut else (var + eps).rsqrt()
    rc = bc(rstd)
    xh = d * rc[:, None]
    one = torch.ones(C, dtype=x.dtype, device=x.device)
    ga = one if gamma is None else gamma.to(x)
    be = torch.zeros_like(one) if beta is None else beta.to(x)
    sc = torch.ones(N, C, dtype=x.dtype, device=x.device) if cs is None else cs.to(x)
    sh = torch.zeros_like(sc) if csh is None else csh.to(x)
    if 'beta_unscaled' in mut:
        pre = xh * (ga * sc)[:, None] + (be + sh)[:, None]
    else:
        pre = (xh * ga + be) * sc[:, None] + sh[:, None]
    slope = 0.2 if 'slope' in mut else LEAKY
    r = {'oh': oh, 'cnt': cnt, 'mean': mean, 'var': var, 'rstd': rstd, 'xh': xh, 'pre': pre, 'ga': ga, 'be': be,
         'sc': sc, 'sh': sh, 'A': rc * ga * sc, 'B': (be - bc(mean) * rc * ga) * sc + sh,
         'y': act_fwd(pre, act, slope, 'sigmoid' in mut), 'sums': torch.stack((gs(x.sum(1)), gs((x * x).sum(1))), -1)}
    if dy is None:
        return r
    dpre = dy * act_grad(pre, act, slope)
    gp = ga * sc
    t1, t2 = dpre.sum(1), (dpre * xh).sum(1)
    m1, m2 = gs(gp * t1) / cnt, gs(gp * t2) / cnt      # mean_g(d^), mean_g(d^ x^)
    Q = -rstd * rstd * m2
    R = rstd * rstd * mean * m2 - rstd * m1
    dh = dpre * gp[:, None]
    dx = rc[:, None] * (dh - bc(m1)[:, None] - xh * bc(m2)[:, None])  # = A dpre + Q x + R
    if 'no_Q' in mut:
        dx = r['A'][:, None] * dpre + bc(R)[:, None]
    if 'no_R' in mut:
        dx = r['A'][:, None] * dpre + bc(Q)[:, None] * x
    colsum = dx.sum((0, 1))
    if add is not None:
        dx = dx + add
        if 'colsum_before_add' not in mut:
            colsum = dx.sum((0, 1))
    dgamma = (sc * ((dpre * x).sum(1) * rc if 'dgamma_no_mean' in mut else t2)).sum(0)
    dscale = ga * t2 if 'dscale_no_beta' in mut else ga * t2 + be * t1
    r.update(dpre=dpre, S=torch.stack((t1, (dpre * x).sum(1)), -1), t1=t1, t2=t2, m1=m1, m2=m2, Q=Q, R=R, dx=dx,
             colsum=colsum, dgamma=dgamma, dbeta=(sc * t1).sum(0), dscale=dscale, dshift=t1)
    return r


def gn_expect(x, G, eps, act, lay, gamma=None, beta=None, cs=None, csh=None, dy=None, add=None, init=None, ecs=None,
              ecsh=None):
    """{output: (reference, tolerance)} of the GroupNorm kernels fed these exact inputs (x, dy, add: float64 [N, V, C]
    of bf16 values). `lay`: sum lengths from `layout`. `init`: the starting values of the accumulated outputs
    (dgamma, dbeta, colsum). ecs / ecsh: bounds of cond_scale / cond_shift when those are themselves computed.

    Statistics: fp32 per-thread sums of Ls terms, fp64 combine: |err| <= gam(Ls) sum|x| (and sum x^2). mean and var
    are formed in fp64 from those sums (var = ss/n - mean^2), rstd = 1/sqrt(var + eps) in fp64, then rounded to fp32:
    rel. error rel_r = q/(1 - q) + F32 with q = err(var)/(var + eps).
    Coefficients: A = rstd gamma s and B = (beta - mu rstd gamma) s + a, each product and sum rounded in fp32;
    pre = fma(x, A, B): |err| <= |x| err(A) + err(B) + F32 |pre|.
    Activation: identity, ReLU, LeakyReLU are 1-Lipschitz in pre; SiLU is 1.1-Lipschitz, plus the tanh.approx error:
    silu = h (1 + t) with h = pre/2, so |pre|/2 * ETANH |t|. Output rounding: U |y| (bf16).
    Backward: dpre = dy act'(pre). SiLU: |silu''| <= 1/2 times the pre error, plus (1/2) ETANH |t| |1 - pre t| from
    the tanh (d silu' / dt), plus a few fp32 roundings. ReLU / LeakyReLU: an element whose pre lies within its own
    bound of 0 may take either slope: its dpre bound is |dy| (1 - slope) there.
    S = fp32 sums of Lr terms of dpre and dpre x. T2 = rstd (S2 - mu S1), m1 / m2 = fp64 sums of fp32 products,
    Q = -rstd^2 m2, R = rstd (m2 rstd mu - m1); dx = A dpre + Q x + R (+ add): the bounds of A, Q, R times the
    magnitudes they multiply, three fp32 roundings, and the bf16 rounding. dgamma / dbeta sum N fp32 terms into the
    caller's values; dx_colsum sums the fp32 dx over Lc terms into the caller's values."""
    r = gn_ref(x, G, eps, act, gamma, beta, cs, csh, dy, add)
    N, V, C = x.shape
    oh, cnt = r['oh'], r['cnt']
    gs = lambda t: t @ oh
    bc = lambda t: t @ oh.T
    ax = x.abs()
    sx, sxx = gs(ax.sum(1)), gs((x * x).sum(1))
    es, ess = (gam(lay['Ls']) + F64) * sx, (gam(lay['Ls']) + F64) * sxx
    mean, var, rstd = r['mean'], r['var'], r['rstd']
    emean = es / cnt
    emu = emean + F32 * mean.abs()
    evar = ess / cnt + (2 * mean.abs() + emean) * emean + F64 * (sxx / cnt + mean * mean)
    q = evar / (var + eps)
    assert float(q.max()) < 0.5, 'statistics too imprecise for the linearised rstd bound'
    rel_r = q / (1 - q) + F32
    rc, mc, emuc, relc = bc(rstd), bc(mean), bc(emu), bc(rel_r)
    ga, be, sc, sh = r['ga'], r['be'], r['sc'], r['sh']
    A, Bv = r['A'], r['B']
    m = mc * rc * ga
    eA = A.abs() * (relc + 3 * F32)
    em = rc * ga.abs() * emuc + m.abs() * (relc + 2 * F32)
    eB = sc.abs() * (em + F32 * (be - m).abs()) + F32 * ((be - m) * sc).abs() + F32 * Bv.abs()
    if ecs is not None:
        eA = eA + rc * ga.abs() * ecs
        eB = eB + (be - m).abs() * ecs
    if ecsh is not None:
        eB = eB + ecsh
    pre, y = r['pre'], r['y']
    epre = ax * eA[:, None] + eB[:, None] + F32 * pre.abs()
    t = torch.tanh(pre / 2)
    if act == 1:
        ey = 1.1 * epre + 0.5 * pre.abs() * ETANH * t.abs() + 3 * F32 * y.abs()
    elif act == 2:
        ey = epre + F32 * y.abs()
    else:
        ey = epre
    tol = lambda e: SLACK * e + TINY
    out = {'sums': (r['sums'], tol(torch.stack((es, ess), -1))),
           'A': (A, tol(eA)), 'B': (Bv, tol(eB)),
           'mean_rstd': (torch.stack((mean, rstd), -1), tol(torch.stack((emu, rel_r * rstd), -1))),
           'y': (y, tol(ey + U * y.abs()))}
    r['kink'] = (pre.abs() <= epre) if act in (2, 3) else torch.zeros_like(pre, dtype=torch.bool)
    if dy is None:
        return out, r
    dpre, ad = r['dpre'], dy.abs()
    if act == 1:
        edpre = ad * (0.5 * epre + 0.5 * ETANH * t.abs() * (1 - pre * t).abs() + 3 * F32 * (1 + pre.abs())) \
            + F32 * dpre.abs()
    elif act in (2, 3):
        jump = 1 - LEAKY if act == 2 else 1.0
        edpre = torch.where(r['kink'], ad * jump, torch.zeros_like(ad)) + F32 * dpre.abs()
    else:
        edpre = torch.zeros_like(dpre)
    eS1 = edpre.sum(1) + gam(lay['Lr']) * dpre.abs().sum(1)
    eS2 = (edpre * ax).sum(1) + gam(lay['Lr']) * (dpre * x).abs().sum(1)
    S1, S2 = r['S'][..., 0], r['S'][..., 1]
    t1, t2 = r['t1'], r['t2']
    et1 = eS1
    et2 = rc * (eS2 + mc.abs() * eS1 + emuc * S1.abs()) + relc * t2.abs() + 3 * F32 * rc * (S2.abs() + (mc * S1).abs())
    gp = ga * sc
    egp = F32 * gp.abs() + (ga.abs() * ecs if ecs is not None else 0)
    m1, m2 = r['m1'], r['m2']
    em1 = gs(gp.abs() * et1 + egp * t1.abs() + 2 * F32 * (gp * t1).abs()) / cnt + F32 * m1.abs()
    em2 = gs(gp.abs() * et2 + egp * t2.abs() + 2 * F32 * (gp * t2).abs()) / cnt + F32 * m2.abs()
    Q, R = r['Q'], r['R']
    eQ = rstd * rstd * em2 + Q.abs() * (2 * rel_r + 2 * F32)
    eR = rstd * (rstd * m2.abs() * emu + rstd * (mean * m2).abs() * rel_r + rstd * mean.abs() * em2 + em1
                 + 3 * F32 * (rstd * (m2 * mean).abs() + m1.abs())) + R.abs() * (rel_r + F32)
    Qc, Rc, eQc, eRc = bc(Q), bc(R), bc(eQ), bc(eR)
    adda = add.abs() if add is not None else 0
    edx = (A.abs() + eA)[:, None] * edpre + eA[:, None] * dpre.abs() + eQc[:, None] * ax + eRc[:, None] \
        + 3 * F32 * ((A[:, None] * dpre).abs() + (Qc[:, None] * x).abs() + Rc.abs()[:, None] + adda)
    dx = r['dx']
    init = init or {}
    z = torch.zeros(C, dtype=x.dtype, device=x.device)
    ig, ib, icol = (init.get(k, z).to(x) for k in ('dgamma', 'dbeta', 'colsum'))
    esc = ecs if ecs is not None else 0
    out.update({
        'S': (r['S'], tol(torch.stack((eS1, eS2), -1))),
        'Q': (Qc, tol(eQc)), 'R': (Rc, tol(eRc)),
        'dx': (dx, tol(edx + U * dx.abs())),
        'dgamma': (ig + r['dgamma'], tol((sc.abs() * et2 + esc * t2.abs()).sum(0)
                                         + gam(N + 2) * (ig.abs() + (sc * t2).abs().sum(0)))),
        'dbeta': (ib + r['dbeta'], tol((sc.abs() * et1 + esc * t1.abs()).sum(0)
                                       + gam(N + 2) * (ib.abs() + (sc * t1).abs().sum(0)))),
        'dcond_scale': (r['dscale'], tol(ga.abs() * et2 + be.abs() * et1 + 2 * F32 * ((ga * t2).abs() + (be * t1).abs()))),
        'dcond_shift': (r['dshift'], tol(et1)),
        'dx_colsum': (icol + r['colsum'], tol(edx.sum((0, 1)) + gam(lay['Lc']) * (icol.abs() + dx.abs().sum((0, 1))))),
    })
    r['edpre'] = edpre
    return out, r


def adagn_expect(cond, ws, bs=None, wa=None, ba=None, dscale=None, dshift=None, cbar=None, dv=True, edscale=None,
                 edshift=None):
    """{output: (reference, tolerance)} of og_adagn_cond_fwd / _bwd. cond: float64 [N, V, D]; ws, wa: [C, D].
    The backward is checked on the inputs it is given (dscale, dshift, and the forward's fp32 cbar).
    Forward: cbar = fp32 sums of ceil(V / lanes) terms per thread and `lanes` = 256 // D per channel, then / V; scale
    and shift are fma chains of D terms. Backward: dW, db sum N fp32 terms; dcond sums 2 ceil(C / 32) terms per lane
    and 5 shuffle steps, then / V. edscale / edshift: bounds of dscale / dshift when they are themselves computed."""
    N, V, D = cond.shape
    C = ws.shape[0]
    lanes = 256 // D
    cb = cond.sum(1) / V if dv else cond.sum(1)
    ecb = gam(-(-V // lanes) + lanes + 2) * cond.abs().sum(1) / V
    zc = torch.zeros(C, dtype=cond.dtype, device=cond.device)
    bs_, ba_ = (zc if b is None else b.to(cond) for b in (bs, ba))
    ws = ws.to(cond)
    tol = lambda e: SLACK * e + TINY
    out = {'cbar': (cb, tol(ecb)),
           'scale': (cb @ ws.T + bs_, tol(gam(D + 2) * (bs_.abs() + cb.abs() @ ws.abs().T) + ecb @ ws.abs().T))}
    if wa is not None:
        wa = wa.to(cond)
        out['shift'] = (cb @ wa.T + ba_, tol(gam(D + 2) * (ba_.abs() + cb.abs() @ wa.abs().T) + ecb @ wa.abs().T))
    if dscale is None:
        return out
    ds, cbk = dscale.to(cond), cbar.to(cond)
    eds = edscale if edscale is not None else torch.zeros_like(ds)
    out['dw_scale'] = (ds.T @ cbk, tol(eds.T @ cbk.abs() + gam(N + 2) * (ds.abs().T @ cbk.abs())))
    out['db_scale'] = (ds.sum(0), tol(eds.sum(0) + gam(N + 2) * ds.abs().sum(0)))
    g = ds @ ws
    eg = eds @ ws.abs() + gam(2 * -(-C // 32) + 8) * (ds.abs() @ ws.abs())
    if dshift is not None:
        dh = dshift.to(cond)
        edh = edshift if edshift is not None else torch.zeros_like(dh)
        out['dw_shift'] = (dh.T @ cbk, tol(edh.T @ cbk.abs() + gam(N + 2) * (dh.abs().T @ cbk.abs())))
        out['db_shift'] = (dh.sum(0), tol(edh.sum(0) + gam(N + 2) * dh.abs().sum(0)))
        if wa is not None:
            g = g + dh @ wa
            eg = eg + edh @ wa.abs() + gam(2 * -(-C // 32) + 8) * (dh.abs() @ wa.abs())
    div = V if dv else 1
    out['dcond'] = ((g / div)[:, None].expand(N, V, D), tol((eg / V + F32 * (g / V).abs())[:, None].expand(N, V, D)))
    return out


def check(name, got, ref, tol):
    got = got.double().to(ref.device)
    assert got.shape == ref.shape, f'{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
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


def bf16_ulps(got, ref):
    """|got - ref| in units of the bf16 spacing at |ref| (2^(e - 7) for ref in [2^e, 2^(e+1)))."""
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126)))
    return (got.double() - ref).abs() / torch.exp2(e - 7)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference against PyTorch, and the tolerances reject the mistakes they exist to catch
# ------------------------------------------------------------------------------------------------------------------
def _cpu_rand(shape, seed, amp=1.0, off=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * amp + off).to(BF16).double()


@pytest.mark.parametrize('act', [0, 1, 2, 3])
@pytest.mark.parametrize('G,cond', [(1, False), (4, True), (8, False)])
def test_reference_matches_pytorch(G, cond, act):
    """gn_ref against F.group_norm, the activation modules and autograd, in float64."""
    N, V, C = 2, 12, 16
    x, dy = _cpu_rand((N, V, C), 1, 1.5, 0.4), _cpu_rand((N, V, C), 2)
    gamma, beta = 1 + 0.3 * _cpu_rand((C,), 3), 0.3 * _cpu_rand((C,), 4)
    cs, csh = (1 + 0.3 * _cpu_rand((N, C), 5), 0.3 * _cpu_rand((N, C), 6)) if cond else (None, None)
    r = gn_ref(x, G, 1e-5, act, gamma, beta, cs, csh, dy)
    xt, gt, bt = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    cst = cs.clone().requires_grad_(True) if cond else None
    csht = csh.clone().requires_grad_(True) if cond else None
    h = F.group_norm(xt.permute(0, 2, 1), G, gt, bt, 1e-5).permute(0, 2, 1)
    if cond:
        h = h * cst[:, None] + csht[:, None]
    y = [lambda v: v, F.silu, lambda v: F.leaky_relu(v, LEAKY), F.relu][act](h)
    y.backward(dy)
    torch.testing.assert_close(r['y'], y.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r['dx'], xt.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(r['dgamma'], gt.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(r['dbeta'], bt.grad, rtol=1e-10, atol=1e-10)
    if cond:
        torch.testing.assert_close(r['dscale'], cst.grad, rtol=1e-10, atol=1e-10)
        torch.testing.assert_close(r['dshift'], csht.grad, rtol=1e-10, atol=1e-10)
    # dx = A dpre + Q x + R, the form the kernels evaluate
    bc = lambda t: t @ r['oh'].T
    torch.testing.assert_close(r['dx'], r['A'][:, None] * r['dpre'] + bc(r['Q'])[:, None] * x + bc(r['R'])[:, None],
                               rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(r['y'], act_fwd(x * r['A'][:, None] + r['B'][:, None], act), rtol=1e-10, atol=1e-10)


def test_adagn_reference_matches_pytorch():
    N, V, D, C = 2, 10, 6, 16
    cond = _cpu_rand((N, V, D), 10)
    ws, bs, wa, ba = _cpu_rand((C, D), 11), _cpu_rand((C,), 12), _cpu_rand((C, D), 13), _cpu_rand((C,), 14)
    ds, dh = _cpu_rand((N, C), 15), _cpu_rand((N, C), 16)
    ct = cond.clone().requires_grad_(True)
    p = [t.clone().requires_grad_(True) for t in (ws, bs, wa, ba)]
    cb = ct.mean(1)
    (F.linear(cb, p[0], p[1]) * ds + F.linear(cb, p[2], p[3]) * dh).sum().backward()
    ex = adagn_expect(cond, ws, bs, wa, ba, ds, dh, cb.detach())
    torch.testing.assert_close(ex['scale'][0], F.linear(cb, ws, bs).detach())
    torch.testing.assert_close(ex['dcond'][0], ct.grad)
    for name, t in zip(('dw_scale', 'db_scale', 'dw_shift', 'db_shift'), p):
        torch.testing.assert_close(ex[name][0], t.grad)


def _rejects(got, expect):
    with pytest.raises(AssertionError):
        check_all(got, expect)


def _exact(ex):
    """A kernel that is exactly right: the reference rounded as each output is stored."""
    return {n: (v[0].to(BF16).double() if n in ('y', 'dx') else v[0].float().double()) for n, v in ex.items()}


def _mut(x, G, act, kw, mut):
    return gn_ref(x, G, 1e-5, act, mut=mut, **kw)


def test_tolerances_reject_plausible_bugs_forward():
    N, V, C, G = 2, 1, 16, 2          # V * C/G = 8 elements per group: the unbiased variance is visible
    x = _cpu_rand((N, V, C), 20, 1.0, 0.5)
    kw = dict(gamma=1 + 0.3 * _cpu_rand((C,), 21), beta=0.5 + 0.3 * _cpu_rand((C,), 22),
              cs=1.5 + 0.3 * _cpu_rand((N, C), 23), csh=0.3 * _cpu_rand((N, C), 24))
    for act in (0, 1, 2, 3):
        ex, _ = gn_expect(x, G, 1e-5, act, layout(N, V, C), **kw)
        exact = _exact(ex)
        check_all({k: exact[k] for k in ('y', 'A', 'B', 'mean_rstd')}, ex)
        for mut in ('unbiased', 'group_shift', 'beta_unscaled'):
            _rejects({'y': _mut(x, G, act, kw, (mut,))['y'].to(BF16).double()}, ex)
    # LeakyReLU slope 0.2; SiLU replaced by the sigmoid (on inputs with negative pre-activations)
    ex, _ = gn_expect(x, G, 1e-5, 2, layout(N, V, C), **kw)
    _rejects({'y': _mut(x, G, 2, kw, ('slope',))['y'].to(BF16).double()}, ex)
    ex, _ = gn_expect(x, G, 1e-5, 1, layout(N, V, C), **kw)
    _rejects({'y': _mut(x, G, 1, kw, ('sigmoid',))['y'].to(BF16).double()}, ex)
    # eps outside the square root, on a constant group (var = 0)
    xc = x.clone()
    xc[0, :, :C // G] = 0.75
    ex, _ = gn_expect(xc, G, 1e-5, 0, layout(N, V, C), **kw)
    check_all({'mean_rstd': _exact(ex)['mean_rstd']}, ex)
    bad = _mut(xc, G, 0, kw, ('eps_outside',))
    _rejects({'mean_rstd': torch.stack((bad['mean'], bad['rstd']), -1).float().double()}, ex)


def test_tolerances_reject_plausible_bugs_backward():
    N, V, C, G = 3, 24, 16, 2
    x = _cpu_rand((N, V, C), 30, 1.0, 0.8)
    dy, add = _cpu_rand((N, V, C), 31), _cpu_rand((N, V, C), 32)
    kw = dict(gamma=1 + 0.3 * _cpu_rand((C,), 33), beta=0.5 + 0.3 * _cpu_rand((C,), 34),
              cs=1.5 + 0.3 * _cpu_rand((N, C), 35), csh=0.3 * _cpu_rand((N, C), 36), dy=dy, add=add)
    init = {k: _cpu_rand((C,), 37 + i).float() for i, k in enumerate(('dgamma', 'dbeta', 'colsum'))}
    for act in (0, 1, 2, 3):
        ex, r = gn_expect(x, G, 1e-5, act, layout(N, V, C, None, None, True), init=init, **kw)
        exact = _exact(ex)
        check_all({k: exact[k] for k in ('dx', 'S', 'Q', 'R', 'dgamma', 'dbeta', 'dcond_scale', 'dcond_shift',
                                         'dx_colsum')}, ex)
        mutated = lambda m: _mut(x, G, act, kw, (m,))
        _rejects({'dx': mutated('no_Q')['dx'].to(BF16).double()}, ex)
        _rejects({'dx': mutated('no_R')['dx'].to(BF16).double()}, ex)
        _rejects({'dgamma': (init['dgamma'] + mutated('dgamma_no_mean')['dgamma']).float().double()}, ex)
        _rejects({'dcond_scale': mutated('dscale_no_beta')['dscale'].float().double()}, ex)
        _rejects({'dx_colsum': (init['colsum'] + mutated('colsum_before_add')['colsum']).float().double()}, ex)
        # accumulated outputs overwritten instead of accumulated
        _rejects({'dbeta': r['dbeta'].float().double()}, ex)


def test_tolerance_rejects_undivided_dcond():
    N, V, D, C = 2, 7, 6, 40
    cond = _cpu_rand((N, V, D), 40)
    ws, wa = _cpu_rand((C, D), 41), _cpu_rand((C, D), 42)
    ds, dh = _cpu_rand((N, C), 43), _cpu_rand((N, C), 44)
    cb = cond.mean(1).float().double()
    ex = adagn_expect(cond, ws, None, wa, None, ds, dh, cb)
    check_all({k: v[0].float().double() for k, v in ex.items()}, ex)
    bad = adagn_expect(cond, ws, None, wa, None, ds, dh, cb, dv=False)
    _rejects({'dcond': bad['dcond'][0].float().double()}, ex)
    _rejects({'cbar': bad['cbar'][0].float().double()}, ex)


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation of the GroupNorm entry points (no device needed)
# ------------------------------------------------------------------------------------------------------------------
def test_norm_act_argument_validation_returns_status_codes():
    import ctypes
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error())
    # C % 8 != 0
    bad(lib.og_gn_stats(p, 1, 16, 12, 1, p, None), b'C%8==0')
    bad(lib.og_gn_act_fwd(p, p, None, None, None, None, 1e-5, 1, 0, p, p, p, p, 1, 16, 12, None), b'C%8==0')
    bad(lib.og_affine_act_fwd(p, p, p, p, 1, 16, 12, 0, None), b'multiple of 8')
    bad(lib.og_affine_act_bwd_apply(p, p, p, p, None, None, None, p, 0, 1, 16, 12, None), b'multiple of 8')
    # G > 64, and C not a multiple of G
    bad(lib.og_gn_stats(p, 1, 16, 1024, 128, p, None), b'G<=64')
    bad(lib.og_gn_finalize(p, 1, 1024, 128, 16, 1e-5, None, None, None, None, p, p, p, None), b'G<=64')
    bad(lib.og_gn_finalize(p, 1, 96, 64, 16, 1e-5, None, None, None, None, p, p, p, None), b'C%G==0')
    bad(lib.og_gn_bwd_finalize(p, p, None, None, None, 1, 1024, 128, 16, p, p, None, None, None, None, None), b'G<=64')
    bad(lib.og_gn_act_fwd(p, p, None, None, None, None, 1e-5, 128, 0, p, p, p, p, 1, 16, 1024, None), b'G<=64')
    bad(lib.og_gn_act_bwd(p, p, p, p, p, p, None, None, None, 128, 0, None, p, None, None, None, None, None, 1, 16,
                          1024, None, 0, None), b'G<=64')
    bad(lib.og_gn_stats(p, 1, 16, 40, 3, p, None), b'C%G==0')
    # C > 2048
    bad(lib.og_gn_stats(p, 1, 16, 4096, 1, p, None), b'> 2048')
    bad(lib.og_affine_act_bwd_reduce(p, p, p, p, 0, p, 1, 16, 4096, None, 0, None), b'<= 2048')
    # dx_colsum over N > 1 samples without a workspace
    bad(lib.og_gn_act_bwd(p, p, p, p, p, p, None, None, None, 1, 0, None, p, None, None, None, None, p, 2, 16, 64,
                          None, 0, None), b'workspace')
    # Q without R; S without mean_rstd
    bad(lib.og_affine_act_bwd_apply(p, p, p, p, p, None, None, p, 0, 1, 16, 64, None), b'Q and R')
    bad(lib.og_gn_act_bwd(p, p, p, p, p, None, None, None, None, 1, 0, None, p, None, None, None, None, None, 1, 16, 64,
                          None, 0, None), b'S and mean_rstd')
    # activation code 4, on every entry point that takes one
    bad(lib.og_affine_act_fwd(p, p, p, p, 1, 16, 64, 4, None), b'activation code 4')
    bad(lib.og_affine_act_bwd_apply(p, p, p, p, None, None, None, p, 4, 1, 16, 64, None), b'activation code 4')
    bad(lib.og_affine_act_bwd_reduce(p, p, p, p, 4, p, 1, 16, 64, None, 0, None), b'activation code 4')
    bad(lib.og_gn_act_fwd(p, p, None, None, None, None, 1e-5, 1, 4, p, p, p, p, 1, 16, 64, None), b'activation code 4')
    bad(lib.og_gn_act_bwd(p, p, p, p, None, None, None, None, None, 1, 4, None, p, None, None, None, None, None, 1, 16,
                          64, None, 0, None), b'activation code 4')
    # D outside [1, 64] in the AdaGN conditioning
    bad(lib.og_adagn_cond_fwd(p, 1, 16, 65, p, None, None, None, 64, p, p, None, None), b'dim_cond=65')
    bad(lib.og_adagn_cond_bwd(p, None, p, p, None, 1, 16, 0, 64, p, None, None, None, None, None), b'dim_cond=0')


def test_layout_mirror_covers_every_branch():
    """The cases below reach each launch branch: this pins the geometry mirror on the H100's 132 SMs."""
    if torch.cuda.is_available() and num_sms() != 132:
        pytest.skip('the branch table is worked out for 132 SMs')
    C, N, V = 128, 2, 4096
    assert not layout(N, V, C, ws_reduce=None)['reduce_partials']
    assert not layout(N, V, C, ws_reduce=4 * (N * 2 * C - 1))['reduce_partials']
    lay = layout(N, V, C, ws_reduce=4 * 3 * N * 2 * C)
    assert lay['reduce_partials'] and lay['gr'] == 3
    assert layout(N, V, C, ws_reduce=64 << 20)['gr'] > 3
    assert not layout(1, V, C, colsum=True, ws_bwd=None)['bwd_partials']
    lay = layout(N, V, C, colsum=True, ws_bwd=4 * N * C)
    assert lay['bwd_partials'] and lay['gb'] == 1
    assert 1 < layout(N, V, C, colsum=True, ws_bwd=4 * 5 * N * C)['gb'] < layout(N, V, C, colsum=True,
                                                                                  ws_bwd=64 << 20)['gb']
    assert reduce_grid(300, 15, 6) == (1, 16)      # one block per sample


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _count():
    from open_genie_b200 import _lib
    torch.cuda.synchronize()
    return _lib.launch_count()


def _rand(shape, seed, amp=1.0, off=0.0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * amp + off).to(dtype)


def _ptr(t):
    return None if t is None else (t.ptr() if isinstance(t, Guarded) else t.data_ptr())


_WS = {}


def workspace(nbytes):
    """(pointer, bytes) of an fp32 scratch buffer of nbytes (None for 0)."""
    if not nbytes:
        return None, 0
    if nbytes not in _WS:
        _WS[nbytes] = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    return _WS[nbytes].data_ptr(), nbytes


BIG_WS = 64 << 20
BWD_OUTS = ('dgamma', 'dbeta', 'dcond_scale', 'dcond_shift', 'add', 'dx_colsum')
# observations gathered while the tests run (reported by the PR, not asserted): max SiLU error in bf16 ulps per form,
# and which outputs the one- and two-launch forms produce bit-identically
OBSERVED = {'silu_ulps': {}, 'bit_equal': {}, 'var_rel_err': {}}


def chain_run(N, V, C, G, act, seed, *, affine=True, cond=False, shift=True, amp=1.0, off=0.0, chan_amp=1.0, eps=1e-5,
              ws_reduce=BIG_WS, ws_bwd=BIG_WS, drop=(), forms=('one', 'two'), backward=True):
    """Runs statistics -> forward (both forms) -> backward reduction -> backward (both forms) on guarded outputs and
    checks every output and launch count against `gn_expect`. Returns (expect, reference, outputs)."""
    assert C % G == 0
    if (C // G) % 8:
        forms = tuple(f for f in forms if f == 'two')
    x = _rand((N, V, C), seed, amp) + _rand((1, 1, C), seed + 1, chan_amp, off)
    x = x.to(BF16)
    gamma = (1 + 0.3 * _rand((C,), seed + 2, dtype=F32T)) if affine else None
    beta = (0.3 * _rand((C,), seed + 3, dtype=F32T)) if affine else None
    cs = (1 + 0.3 * _rand((N, C), seed + 4, dtype=F32T)) if cond else None
    csh = (0.3 * _rand((N, C), seed + 5, dtype=F32T)) if (cond and shift) else None
    dy, add = _rand((N, V, C), seed + 6), _rand((N, V, C), seed + 7)
    use_add = 'add' not in drop
    colsum = 'dx_colsum' not in drop
    init = {k: _rand((C,), seed + 8 + i, dtype=F32T) for i, k in enumerate(('dgamma', 'dbeta', 'colsum'))}
    lay = layout(N, V, C, ws_reduce, ws_bwd, colsum)
    xd = x.double()
    ex, ref = gn_expect(xd, G, eps, act, lay, gamma, beta, cs, csh, dy.double() if backward else None,
                        add.double() if use_add else None, init)
    got = {}
    # statistics: the caller zeroes the sums
    sums = Guarded((N, G, 2), F64T, init=torch.zeros(N, G, 2))
    n0 = _count()
    _call('og_gn_stats', x.data_ptr(), N, V, C, G, sums.ptr())
    assert _count() - n0 == 1
    check('sums', sums.t, *ex['sums'])
    sums.check_guard('sums')
    got['sums'] = sums.t
    got['_in'] = dict(x=x, dy=dy, add=add, gamma=gamma, beta=beta, cs=cs)
    fw = {}
    for form in forms:
        A, B, mr, y = Guarded((N, C), F32T), Guarded((N, C), F32T), Guarded((N, G, 2), F32T), Guarded((N, V, C), BF16)
        n0 = _count()
        if form == 'one':
            _call('og_gn_act_fwd', x.data_ptr(), sums.ptr(), _ptr(gamma), _ptr(beta), _ptr(cs), _ptr(csh), eps, G, act,
                  y.ptr(), A.ptr(), B.ptr(), mr.ptr(), N, V, C)
            assert _count() - n0 == 1
        else:
            _call('og_gn_finalize', sums.ptr(), N, C, G, V, eps, _ptr(gamma), _ptr(beta), _ptr(cs), _ptr(csh), A.ptr(),
                  B.ptr(), mr.ptr())
            _call('og_affine_act_fwd', x.data_ptr(), A.ptr(), B.ptr(), y.ptr(), N, V, C, act)
            assert _count() - n0 == 2
        torch.cuda.synchronize()
        outs = {'A': A, 'B': B, 'mean_rstd': mr, 'y': y}
        check_all({n: o.t for n, o in outs.items()}, ex)
        for n, o in outs.items():
            o.check_guard(f'{form}:{n}')
        fw[form] = outs
        if act == 1:
            u = float(bf16_ulps(y.t, ex['y'][0]).max())
            OBSERVED['silu_ulps'][f'fwd_{form}'] = max(OBSERVED['silu_ulps'].get(f'fwd_{form}', 0.0), u)
    if len(fw) == 2:
        _note_equal(fw, ('A', 'B', 'mean_rstd', 'y'), act)
    got.update({f'{f}:{n}': o.t for f, outs in fw.items() for n, o in outs.items()})
    if act in (2, 3):       # the kink allowance must stay the exception
        assert float(ref['kink'].double().mean()) < 1e-3, 'too many pre-activations within their bound of 0'
    if not backward:
        return ex, ref, got
    A, B, mr = (fw[forms[0]][n] for n in ('A', 'B', 'mean_rstd'))
    # backward reduction: S zeroed by the caller
    S = Guarded((N, C, 2), F32T, init=torch.zeros(N, C, 2))
    wp, wb = workspace(ws_reduce)
    n0 = _count()
    _call('og_affine_act_bwd_reduce', dy.data_ptr(), x.data_ptr(), A.ptr(), B.ptr(), act, S.ptr(), N, V, C, wp, wb)
    assert _count() - n0 == 1 + lay['reduce_partials'], 'og_sum_partials ran (or not) against the launch rule'
    check('S', S.t, *ex['S'])
    S.check_guard('S')
    got['S'] = S.t
    bw = {}
    for form in forms:
        o = {'dx': Guarded((N, V, C), BF16)}
        if 'dgamma' not in drop:
            o['dgamma'] = Guarded((C,), F32T, init=init['dgamma'])
        if 'dbeta' not in drop:
            o['dbeta'] = Guarded((C,), F32T, init=init['dbeta'])
        if 'dcond_scale' not in drop:
            o['dcond_scale'] = Guarded((N, C), F32T)
        if 'dcond_shift' not in drop:
            o['dcond_shift'] = Guarded((N, C), F32T)
        addp = add.data_ptr() if use_add else None
        grads = _ptr(o.get('dgamma')), _ptr(o.get('dbeta')), _ptr(o.get('dcond_scale')), _ptr(o.get('dcond_shift'))
        param = 'dgamma' in o or 'dbeta' in o
        n0 = _count()
        if form == 'one':
            if colsum:
                o['dx_colsum'] = Guarded((C,), F32T, init=init['colsum'])
            wp, wb = workspace(ws_bwd)
            _call('og_gn_act_bwd', dy.data_ptr(), x.data_ptr(), A.ptr(), B.ptr(), S.ptr(), mr.ptr(), _ptr(gamma),
                  _ptr(beta), _ptr(cs), G, act, addp, o['dx'].ptr(), *grads, _ptr(o.get('dx_colsum')), N, V, C, wp, wb)
            assert _count() - n0 == 1 + lay['bwd_partials'] + param, 'og_sum_partials / param_grads launch count'
        else:
            o['Q'], o['R'] = Guarded((N, C), F32T), Guarded((N, C), F32T)
            _call('og_gn_bwd_finalize', S.ptr(), mr.ptr(), _ptr(gamma), _ptr(beta), _ptr(cs), N, C, G, V, o['Q'].ptr(),
                  o['R'].ptr(), *grads)
            _call('og_affine_act_bwd_apply', dy.data_ptr(), x.data_ptr(), A.ptr(), B.ptr(), o['Q'].ptr(), o['R'].ptr(),
                  addp, o['dx'].ptr(), act, N, V, C)
            assert _count() - n0 == 2 + param, 'og_gn_param_grads_kernel launch count'
        torch.cuda.synchronize()
        check_all({n: g.t for n, g in o.items()}, ex)
        for n, g in o.items():
            g.check_guard(f'{form}:{n}')
        bw[form] = o
        got.update({f'{form}:{n}': g.t for n, g in o.items()})
    if len(bw) == 2:
        _note_equal(bw, ('dx', 'dgamma', 'dbeta', 'dcond_scale', 'dcond_shift'), act)
    return ex, ref, got


def _note_equal(by_form, names, act):
    for n in names:
        if n in by_form['one'] and n in by_form['two']:
            a, b = by_form['one'][n].t, by_form['two'][n].t
            ulps = float(bf16_ulps(a, b.double()).max()) if a.dtype == BF16 else 0.0
            k = f'{n}[act {act}]'
            OBSERVED['bit_equal'][k] = max(OBSERVED['bit_equal'].get(k, 0.0), 0.0 if torch.equal(a, b) else max(ulps, 1e-9))


# ------------------------------------------------------------------------------------------------------------------
# statistics: every G, C, V and N value, and (C/G) % 8 != 0
# ------------------------------------------------------------------------------------------------------------------
STATS_CASES = [
    # N, V, C, G
    (1, 1, 8, 1),
    (1, 15, 8, 2),          # C/G = 4: split kernel
    (2, 15, 128, 2),
    (300, 17, 128, 8),      # two blocks per sample
    (300, 15, 512, 64),     # one block per sample
    (2, 256, 192, 8),       # cvs = 24: 16 idle threads per block
    (1, 256, 192, 64),      # C/G = 3, G = 64
    (1, 17, 1536, 2),       # cvs = 192: one row lane, 64 idle threads
    (2, 1, 2048, 8),        # C = 2048: one row lane, every thread busy
    (1, 65536, 2048, 64),
    (2, 65536, 512, 1),
    (1, 256, 40, 5),        # cvs = 5
    (2, 256, 64, 16),       # C/G = 4
    (2, 17, 96, 32),        # C/G = 3
    (1, 65536, 40, 4),      # C/G = 10: vectors cross group boundaries unevenly
    (300, 15, 64, 16),
]


@GPU
@pytest.mark.parametrize('N,V,C,G', STATS_CASES)
def test_stats_and_forward(N, V, C, G):
    """og_gn_stats (both kernels) and both forward forms with SiLU, against float64."""
    chain_run(N, V, C, G, 1, seed=100 + C + G + V % 1000, backward=V * N * C <= (1 << 22))


@GPU
@pytest.mark.parametrize('N,V,C,G', [(2, 4096, 128, 8), (1, 65536, 2048, 64)])
def test_stats_large_mean(N, V, C, G):
    """|mean| = 30 std: the one-pass variance (fp32 per-thread sums of x and x^2, fp64 var = ss/n - mean^2) loses
    precision to cancellation. The derived bound still holds for the statistics, A, B, y and the backward.
    Observed on an H100: with 8 fp32 terms per thread (2 x 4096 x 128) the sums are exact and so is the variance;
    with 768 terms per thread (65536 x 2048, one row lane) the variance is off by up to 0.45 % of the exact value
    (rstd by about 0.23 %, below the bf16 rounding of y)."""
    ex, ref, got = chain_run(N, V, C, G, 1, seed=700, off=30.0, amp=1.0, chan_amp=0.1, backward=N * V * C <= 1 << 22)
    assert float((ref['mean'].abs() / ref['var'].sqrt()).min()) > 25
    s = got['sums'].double()
    cnt = V * C // G
    mean = s[..., 0] / cnt
    var = s[..., 1] / cnt - mean * mean
    OBSERVED['var_rel_err'][(N, V, C, G)] = float(((var - ref['var']).abs() / ref['var']).max())


# ------------------------------------------------------------------------------------------------------------------
# forward and backward, every activation, with and without affine / conditioning, below and above the grid cap
# ------------------------------------------------------------------------------------------------------------------
FWD_VARIANTS = {
    # name: (N, V, C, G, kwargs)
    'affine': (2, 300, 64, 8, dict()),
    'no_affine': (2, 300, 64, 8, dict(affine=False)),
    'cond': (3, 100, 256, 8, dict(cond=True)),
    'cond_scale_only': (3, 100, 256, 1, dict(cond=True, shift=False, affine=False)),
    'beyond_grid_cap': (2, 65536, 128, 8, dict(cond=True)),        # 2 * 65536 * 16 vectors > 132 * 16 * 256
}


@GPU
@pytest.mark.parametrize('act', [0, 1, 2, 3])
@pytest.mark.parametrize('variant', sorted(FWD_VARIANTS))
def test_forward_backward(variant, act):
    N, V, C, G, kw = FWD_VARIANTS[variant]
    if variant == 'beyond_grid_cap':
        assert N * V * C // 8 > num_sms() * 16 * 256
    chain_run(N, V, C, G, act, seed=1000 + 10 * act + len(variant), **kw)


@GPU
@pytest.mark.parametrize('act', [0, 1, 2, 3])
@pytest.mark.parametrize('ws', ['none', 'direct', 'few_blocks', 'full'])
def test_backward_reduce_workspaces(ws, act):
    """og_affine_act_bwd_reduce: no workspace and a workspace of fewer than N * 2C floats add into S directly (one
    block per sample); room for 3 blocks per sample shrinks the grid; 64 MB runs the full grid. All with partials go
    through og_sum_partials (checked by the launch count in chain_run)."""
    N, V, C, G = 2, 4096, 128, 8
    nbytes = {'none': 0, 'direct': 4 * (N * 2 * C - 1), 'few_blocks': 4 * 3 * N * 2 * C, 'full': BIG_WS}[ws]
    chain_run(N, V, C, G, act, seed=2000 + act, ws_reduce=nbytes, forms=('one',))


@GPU
@pytest.mark.parametrize('drop', ['none'] + list(BWD_OUTS))
def test_backward_optional_outputs(drop):
    """Every optional output of the backward given, then each one left out in turn, through both forms."""
    chain_run(2, 520, 128, 8, 1, seed=3000 + len(drop), cond=True, drop=(drop,))


@GPU
@pytest.mark.parametrize('case', ['N1_no_ws', 'exact_NC', 'mid', 'full'])
def test_colsum_workspaces(case):
    """dx_colsum: N = 1 without a workspace (one block adds directly); N > 1 with exactly N * C floats (grid (1, N),
    partials); a mid-size workspace; 64 MB."""
    C, V = 128, 4096
    N = 1 if case == 'N1_no_ws' else 3
    nbytes = {'N1_no_ws': 0, 'exact_NC': 4 * N * C, 'mid': 4 * 7 * N * C, 'full': BIG_WS}[case]
    lay = layout(N, V, C, BIG_WS, nbytes, True)
    assert lay['bwd_partials'] == (case != 'N1_no_ws')
    chain_run(N, V, C, 8, 2, seed=4000 + N, ws_bwd=nbytes, forms=('one',))


@GPU
@pytest.mark.parametrize('act', [0, 1, 2, 3])
def test_pure_activation_backward(act):
    """S = mean_rstd = NULL (og_gn_act_bwd) and Q = R = NULL (og_affine_act_bwd_apply): dx = A dpre (+ add), the
    stand-alone activation's backward. A, B are arbitrary per-(n, c) coefficients here."""
    N, V, C = 2, 777, 64
    x, dy, add = _rand((N, V, C), 5000 + act, 2.0), _rand((N, V, C), 5010), _rand((N, V, C), 5020)
    A, B = _rand((N, C), 5030, 0.5, 1.0, F32T), _rand((N, C), 5040, 0.5, dtype=F32T)
    pre = x.double() * A.double()[:, None] + B.double()[:, None]
    epre = F32 * pre.abs()
    t = torch.tanh(pre / 2)
    dpre = dy.double() * act_grad(pre, act)
    ad = dy.double().abs()
    if act == 1:
        edpre = ad * (0.5 * epre + 0.5 * ETANH * t.abs() * (1 - pre * t).abs() + 3 * F32 * (1 + pre.abs()))
    elif act in (2, 3):
        kink = pre.abs() <= epre
        assert float(kink.double().mean()) < 1e-3
        edpre = torch.where(kink, ad, torch.zeros_like(ad))
    else:
        edpre = torch.zeros_like(ad)
    for use_add in (False, True):
        ref = A.double()[:, None] * dpre + (add.double() if use_add else 0)
        tol = SLACK * (A.double().abs()[:, None] * (edpre + 2 * F32 * dpre.abs()) + F32 * ref.abs() + U * ref.abs()) \
            + TINY
        for form in ('one', 'two'):
            dx = Guarded((N, V, C), BF16)
            addp = add.data_ptr() if use_add else None
            if form == 'one':
                _call('og_gn_act_bwd', dy.data_ptr(), x.data_ptr(), A.data_ptr(), B.data_ptr(), None, None, None, None,
                      None, 1, act, addp, dx.ptr(), None, None, None, None, None, N, V, C, None, 0)
            else:
                _call('og_affine_act_bwd_apply', dy.data_ptr(), x.data_ptr(), A.data_ptr(), B.data_ptr(), None, None,
                      addp, dx.ptr(), act, N, V, C)
            torch.cuda.synchronize()
            check(f'{form}:dx', dx.t, ref, tol)
            dx.check_guard(f'{form}:dx')


@GPU
def test_silu_error_per_element():
    """Every bf16 value in [-40, 40] through SiLU forward (og_affine_act_fwd) and backward (both forms, dy = 1), with
    A = 1, B = 0. The error must stay within the documented tanh.approx bound; the largest error in bf16 ulps is
    recorded (SILU_ULPS in norm_act.cu)."""
    bits = torch.arange(0, 0x7F80, dtype=torch.int16, device=DEV).view(BF16)
    v = bits[(bits.float() <= 40)]
    x = torch.cat((v, -v)).contiguous()
    n = x.numel() // 8 * 8
    x = x[:n].view(1, n // 8, 8).contiguous()
    V = n // 8
    A, B = torch.ones(1, 8, device=DEV), torch.zeros(1, 8, device=DEV)
    xd = x.double()
    t = torch.tanh(xd / 2)
    y_ref, d_ref = act_fwd(xd, 1), act_grad(xd, 1)
    y = Guarded((1, V, 8), BF16)
    _call('og_affine_act_fwd', x.data_ptr(), A.data_ptr(), B.data_ptr(), y.ptr(), 1, V, 8, 1)
    dy = torch.ones_like(x)
    dxs = {}
    for form in ('one', 'two'):
        dx = Guarded((1, V, 8), BF16)
        if form == 'one':
            _call('og_gn_act_bwd', dy.data_ptr(), x.data_ptr(), A.data_ptr(), B.data_ptr(), None, None, None, None, None,
                  1, 1, None, dx.ptr(), None, None, None, None, None, 1, V, 8, None, 0)
        else:
            _call('og_affine_act_bwd_apply', dy.data_ptr(), x.data_ptr(), A.data_ptr(), B.data_ptr(), None, None,
                  None, dx.ptr(), 1, 1, V, 8)
        dxs[form] = dx
    torch.cuda.synchronize()
    ey = 0.5 * xd.abs() * ETANH * t.abs() + 3 * F32 * y_ref.abs()
    check('silu', y.t, y_ref, SLACK * (ey + U * y_ref.abs()) + TINY)
    ed = 0.5 * ETANH * t.abs() * (1 - xd * t).abs() + 4 * F32 * (1 + xd.abs())
    for form, dx in dxs.items():
        check(f'{form}:silu_grad', dx.t, d_ref, SLACK * (ed + U * d_ref.abs()) + TINY)
    OBSERVED['silu_ulps']['sweep_fwd'] = float(bf16_ulps(y.t, y_ref).max())
    for lo, hi in ((-8, 41), (-12, -8), (-17, -12), (-41, -17)):
        sel = (xd >= lo) & (xd < hi)
        OBSERVED['silu_ulps'][f'sweep_fwd[{lo},{hi})'] = float(bf16_ulps(y.t, y_ref)[sel].max())
        for form, dx in dxs.items():
            OBSERVED['silu_ulps'][f'sweep_bwd_{form}[{lo},{hi})'] = float(bf16_ulps(dx.t, d_ref)[sel].max())


# ------------------------------------------------------------------------------------------------------------------
# reproducibility
# ------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize('act', [1, 3])
def test_reductions_are_reproducible(act):
    """Two calls with the same inputs and workspace give bit-identical S, dx, dx_colsum, dgamma and dbeta. Calls with
    different workspace sizes agree within the bound (chain_run checks each against it)."""
    N, V, C, G = 3, 4096, 256, 8
    for ws in (BIG_WS, 4 * 5 * N * 2 * C):
        _, _, got = chain_run(N, V, C, G, act, seed=6000, ws_reduce=ws, ws_bwd=ws, forms=('one',))
        i = got['_in']
        A, B, mr = got['one:A'], got['one:B'], got['one:mean_rstd']
        runs = []
        for _ in range(2):
            S = torch.zeros(N, C, 2, device=DEV)
            o = {'S': S, 'dx': torch.empty_like(i['x']), 'dgamma': torch.ones(C, device=DEV),
                 'dbeta': torch.ones(C, device=DEV), 'dx_colsum': torch.ones(C, device=DEV)}
            wp, wb = workspace(ws)
            _call('og_affine_act_bwd_reduce', i['dy'].data_ptr(), i['x'].data_ptr(), A.data_ptr(), B.data_ptr(), act,
                  S.data_ptr(), N, V, C, wp, wb)
            _call('og_gn_act_bwd', i['dy'].data_ptr(), i['x'].data_ptr(), A.data_ptr(), B.data_ptr(), S.data_ptr(),
                  mr.data_ptr(), i['gamma'].data_ptr(), i['beta'].data_ptr(), None, G, act, i['add'].data_ptr(),
                  o['dx'].data_ptr(), o['dgamma'].data_ptr(), o['dbeta'].data_ptr(), None, None,
                  o['dx_colsum'].data_ptr(), N, V, C, wp, wb)
            runs.append(o)
        torch.cuda.synchronize()
        for n in runs[0]:
            assert torch.equal(runs[0][n], runs[1][n]), (ws, n)


# ------------------------------------------------------------------------------------------------------------------
# AdaGN conditioning
# ------------------------------------------------------------------------------------------------------------------
ADAGN_CASES = [
    # N, V, D, C, shift, bias, dcond
    (2, 1, 1, 40, True, True, True),
    (3, 100, 6, 256, False, False, True),
    (2, 65536, 18, 512, True, True, False),
    (2, 4096, 64, 40, True, False, True),
    (1, 17, 64, 512, False, True, False),
    (2, 2048, 18, 512, True, True, True),       # AdaGN C = 512 at 8 x 16 x 16
    (2, 16384, 18, 256, True, True, True),      # AdaGN C = 256 at 16 x 64 x 64
]


@GPU
@pytest.mark.parametrize('N,V,D,C,shift,bias,dcond', ADAGN_CASES)
def test_adagn_condition(N, V, D, C, shift, bias, dcond):
    seed = 7000 + D + C
    cond = _rand((N, V, D), seed, dtype=F32T)
    ws = _rand((C, D), seed + 1, 0.3, dtype=F32T)
    wa = _rand((C, D), seed + 2, 0.3, dtype=F32T) if shift else None
    bs = _rand((C,), seed + 3, dtype=F32T) if bias else None
    ba = _rand((C,), seed + 4, dtype=F32T) if (bias and shift) else None
    cbar, scale = Guarded((N, D), F32T), Guarded((N, C), F32T)
    sh = Guarded((N, C), F32T) if shift else None
    _call('og_adagn_cond_fwd', cond.data_ptr(), N, V, D, ws.data_ptr(), _ptr(bs), _ptr(wa), _ptr(ba), C, cbar.ptr(),
          scale.ptr(), _ptr(sh))
    torch.cuda.synchronize()
    ex = adagn_expect(cond.double(), ws, bs, wa, ba)
    outs = {'cbar': cbar, 'scale': scale}
    if shift:
        outs['shift'] = sh
    check_all({n: o.t for n, o in outs.items()}, ex)
    ds = _rand((N, C), seed + 5, dtype=F32T)
    dh = _rand((N, C), seed + 6, dtype=F32T) if shift else None
    bo = {'dw_scale': Guarded((C, D), F32T), 'db_scale': Guarded((C,), F32T)}
    if shift:
        bo['dw_shift'], bo['db_shift'] = Guarded((C, D), F32T), Guarded((C,), F32T)
    dc = Guarded((N, V, D), F32T)
    n0 = _count()
    _call('og_adagn_cond_bwd', ds.data_ptr(), _ptr(dh), cbar.ptr(), ws.data_ptr(), _ptr(wa), N, V, D, C,
          bo['dw_scale'].ptr(), bo['db_scale'].ptr(), _ptr(bo.get('dw_shift')), _ptr(bo.get('db_shift')),
          dc.ptr() if dcond else None)
    assert _count() - n0 == 1
    exb = adagn_expect(cond.double(), ws, bs, wa, ba, ds, dh, cbar.t)
    if dcond:
        bo['dcond'] = dc
    else:
        assert dc.untouched(), 'dcond written although NULL was passed'
    check_all({n: o.t for n, o in bo.items()}, exb)
    for n, o in list(outs.items()) + list(bo.items()):
        o.check_guard(n)


# ------------------------------------------------------------------------------------------------------------------
# the product's shapes
# ------------------------------------------------------------------------------------------------------------------
PRODUCT = {
    'gn8_512_4x8x8': (2, 256, 512, 8, dict()),
    'gn8_128_16x64x64_B2': (2, 65536, 128, 8, dict()),
    'gn1_128': (2, 4096, 128, 1, dict()),
    'gn1_256': (2, 2048, 256, 1, dict()),
    'gn1_512': (2, 256, 512, 1, dict()),
    'adagn_512_8x16x16': (2, 2048, 512, 8, dict(cond=True)),
    'adagn_256_16x64x64': (2, 16384, 256, 8, dict(cond=True)),
    'ffn_gn8_512': (2, 1024, 512, 8, dict(affine=True)),        # ST-block FFN: GroupNorm(n_head, 64 n_head)
}


@GPU
@pytest.mark.parametrize('name', sorted(PRODUCT))
def test_product_shapes(name):
    N, V, C, G, kw = PRODUCT[name]
    act = 0 if name.startswith(('adagn', 'ffn')) else 1
    chain_run(N, V, C, G, act, seed=8000 + C + G, **kw)


# ------------------------------------------------------------------------------------------------------------------
# module level: ops.py autograd functions against the float64 emulation (bf16 rounding where the product rounds)
# ------------------------------------------------------------------------------------------------------------------
def _rows(t):
    """Logical (B, C, T, H, W) -> [B, V, C] float64."""
    B, C = t.shape[:2]
    return t.detach().permute(0, 2, 3, 4, 1).reshape(B, -1, C).double()


@GPU
@pytest.mark.parametrize('G,C,act,x_grad', [(8, 128, 'silu', True), (1, 64, 'none', True), (16, 64, 'silu', True),
                                             (32, 96, 'relu', True), (4, 40, 'leaky', True),
                                             (8, 128, 'silu', False), (16, 64, 'none', False)])
def test_group_norm_act_module(G, C, act, x_grad):
    """ops.group_norm_act from fp32 reference-format input: the product rounds x and dy to bf16. (C/G) % 8 == 0 takes
    the one-launch backward, the others (and x without requires_grad) og_gn_bwd_finalize."""
    from open_genie_b200 import ops
    B, T, H, W = 2, 3, 8, 8
    V = T * H * W
    x = (torch.randn(B, C, T, H, W, device=DEV) * 1.3 + 0.2).requires_grad_(x_grad)
    gamma = (1 + 0.3 * torch.randn(C, device=DEV)).requires_grad_(True)
    beta = (0.3 * torch.randn(C, device=DEV)).requires_grad_(True)
    y = ops.group_norm_act(x, gamma, beta, G, 1e-5, act)
    dy = torch.randn(B, C, T, H, W, device=DEV)
    y.backward(dy)
    torch.cuda.synchronize()
    code = ops.act_code(act)
    lay = layout(B, V, C, ops._SCOPE.SCRATCH_BYTES, ops._SCOPE.SCRATCH_BYTES)
    ex, _ = gn_expect(_rows(x.to(BF16)), G, 1e-5, code, lay, gamma.detach(), beta.detach(), dy=_rows(dy.to(BF16)))
    check('y', _rows(y), *ex['y'])
    if x_grad:
        check('dx', _rows(x.grad), *ex['dx'])
    check('dgamma', gamma.grad, *ex['dgamma'])
    check('dbeta', beta.grad, *ex['dbeta'])


@GPU
@pytest.mark.parametrize('act', ['silu', 'leaky', 'relu', 'none'])
def test_activation_module(act):
    """ops.silu and the stand-alone activations (_ActFn) with a scale: y = act(scale x)."""
    from open_genie_b200 import ops
    B, C, T, H, W = 2, 24, 2, 5, 7
    x = torch.randn(B, C, T, H, W, device=DEV, requires_grad=True) * 2
    x.retain_grad()
    scale = 1.0 if act == 'silu' else 0.75
    y = ops.silu(x) if act == 'silu' else ops.activation(x, act, scale)
    dy = torch.randn_like(y)
    y.backward(dy)
    torch.cuda.synchronize()
    code = ops.act_code(act)
    xb, dyb = _rows(x.to(BF16)), _rows(dy.to(BF16))
    pre = xb * scale
    epre = F32 * pre.abs()
    t = torch.tanh(pre / 2)
    yr = act_fwd(pre, code)
    ey = (1.1 * epre + 0.5 * pre.abs() * ETANH * t.abs() + 3 * F32 * yr.abs()) if code == 1 else epre + F32 * yr.abs()
    check('y', _rows(y), yr, SLACK * (ey + U * yr.abs()) + TINY)
    dr = scale * dyb * act_grad(pre, code)
    if code == 1:
        ed = dyb.abs() * (0.5 * epre + 0.5 * ETANH * t.abs() * (1 - pre * t).abs() + 3 * F32 * (1 + pre.abs()))
    elif code in (2, 3):
        kink = pre.abs() <= epre
        ed = torch.where(kink, dyb.abs(), torch.zeros_like(dyb))
    else:
        ed = torch.zeros_like(dyb)
    check('dx', _rows(x.grad), dr, SLACK * (scale * ed + 3 * F32 * dr.abs() + U * dr.abs()) + TINY)


@GPU
def test_adaptive_group_norm_module():
    """AdaptiveGroupNorm: conditioning (fp32 kernels) feeding GroupNorm's cond_scale / cond_shift. The bounds of scale
    and shift enter A, B and the gradients; dcond and the linear weights' gradients are checked through the bounds
    of dscale / dshift."""
    from open_genie_b200.module.norm import AdaptiveGroupNorm
    from open_genie_b200 import ops
    B, D, G, C, T, H, W = 2, 6, 8, 64, 2, 8, 8
    V = T * H * W
    m = AdaptiveGroupNorm(D, G, C).to(DEV)
    torch.manual_seed(0)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn_like(p) * 0.3 + (1.0 if p is m.std.bias or p is m.weight else 0.0))
    x = (torch.randn(B, C, T, H, W, device=DEV) + 0.3).requires_grad_(True)
    cond = torch.randn(B, D, T, 4, 4, device=DEV).requires_grad_(True)
    y = m(x, cond)
    dy = torch.randn_like(y)
    y.backward(dy)
    torch.cuda.synchronize()
    crow = cond.detach().permute(0, 2, 3, 4, 1).reshape(B, -1, D).double()
    exc = adagn_expect(crow, m.std.weight.detach(), m.std.bias.detach(), m.avg.weight.detach(), m.avg.bias.detach())
    cs, ecs = exc['scale'][0], (exc['scale'][1] - TINY) / SLACK
    csh, ecsh = exc['shift'][0], (exc['shift'][1] - TINY) / SLACK
    lay = layout(B, V, C, ops._SCOPE.SCRATCH_BYTES, ops._SCOPE.SCRATCH_BYTES)
    ex, _ = gn_expect(_rows(x.to(BF16)), G, m.eps, 0, lay, m.weight.detach(), m.bias.detach(), cs, csh,
                      dy=_rows(dy.to(BF16)), ecs=ecs, ecsh=ecsh)
    check('y', _rows(y), *ex['y'])
    check('dx', _rows(x.grad), *ex['dx'])
    check('dgamma', m.weight.grad, *ex['dgamma'])
    check('dbeta', m.bias.grad, *ex['dbeta'])
    # dscale = gamma T2 + beta T1 (+ its bound, which includes the effect of the scale's own error through dpre)
    ds, eds = ex['dcond_scale'][0], ex['dcond_scale'][1]
    dh, edh = ex['dcond_shift'][0], ex['dcond_shift'][1]
    cb = crow.sum(1) / crow.shape[1]
    ecb = (exc['cbar'][1] - TINY) / SLACK
    exb = adagn_expect(crow, m.std.weight.detach(), m.std.bias.detach(), m.avg.weight.detach(), m.avg.bias.detach(),
                       ds, dh, cb, edscale=eds, edshift=edh)
    # the kernel multiplies by its own fp32 cbar: add |dscale| err(cbar) to the weight-gradient bounds
    check('std.weight', m.std.weight.grad, exb['dw_scale'][0], exb['dw_scale'][1] + (ds.abs() + eds).T @ ecb)
    check('std.bias', m.std.bias.grad, *exb['db_scale'])
    check('avg.weight', m.avg.weight.grad, exb['dw_shift'][0], exb['dw_shift'][1] + (dh.abs() + edh).T @ ecb)
    check('avg.bias', m.avg.bias.grad, *exb['db_shift'])
    check('dcond', cond.grad.detach().permute(0, 2, 3, 4, 1).reshape(B, -1, D), *exb['dcond'])


@GPU
def test_video_residual_block_with_16_groups():
    """VideoResidualBlock(64, 64, num_groups=16): C/G = 4, so the block takes the unfused path through
    ops.group_norm_act (statistics by the per-channel kernel). Forward and backward against PyTorch in fp32."""
    from open_genie_b200.module.video import VideoResidualBlock
    from helpers import rel_l2
    torch.manual_seed(1)
    blk = VideoResidualBlock(64, 64, num_groups=16).to(DEV)
    with torch.no_grad():
        for name, p in blk.named_parameters():
            if name in ('main.0.weight', 'main.4.weight'):
                p.copy_(1 + 0.3 * torch.randn_like(p))
            else:
                p.copy_(torch.randn_like(p) * (0.05 if p.dim() > 1 else 0.3))
    x = torch.randn(2, 64, 3, 8, 8, device=DEV, requires_grad=True)
    y = blk(x)
    dy = torch.randn_like(y)
    y.backward(dy)
    torch.cuda.synchronize()
    sd = {k: v.detach().float().clone().requires_grad_(True) for k, v in blk.state_dict().items()}
    xr = x.detach().clone().requires_grad_(True)
    g1, g2 = blk.main[0], blk.main[4]

    def conv(h, pre):
        w = sd[pre + '.weight']
        k = w.shape[2:]
        return F.conv3d(h, w, sd[pre + '.bias'], padding=tuple(s // 2 for s in k))
    h = F.silu(F.group_norm(xr, 16, sd['main.0.weight'], sd['main.0.bias'], g1.eps))
    h = conv(h, 'main.2')
    h = F.silu(F.group_norm(h, 16, sd['main.4.weight'], sd['main.4.bias'], g2.eps))
    yr = conv(h, 'main.6') + conv(xr, 'res.1')
    yr.backward(dy)
    assert rel_l2(y.float(), yr.detach()) < 2e-2
    assert rel_l2(x.grad.float(), xr.grad) < 3e-2
    for name, p in blk.named_parameters():
        assert p.grad is not None and rel_l2(p.grad.float(), sd[name].grad) < 3e-2, name


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
def _kernels_run(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


@GPU
def test_dispatch_kernel_names():
    """The chains above reach every kernel of norm_act.cu: each activation's one-launch kernels, the two-launch
    kernels, both statistics kernels, og_sum_partials and og_gn_param_grads."""
    def run():
        for act in range(4):
            chain_run(2, 520, 64, 8, act, seed=9000 + act, ws_reduce=BIG_WS, ws_bwd=BIG_WS)
        chain_run(2, 40, 64, 16, 1, seed=9010)
        test_adagn_condition(2, 10, 6, 40, True, True, True)
    names = _kernels_run(run)
    want = [f'og_gn_act_fwd_kernel<{a}>' for a in range(4)] + \
        [f'og_affine_act_bwd_reduce_kernel<{a}>' for a in range(4)] + \
        [f'og_gn_act_bwd_kernel<{a}>' for a in range(4)] + \
        ['og_sum_partials_kernel', 'og_gn_finalize_kernel', 'og_affine_act_fwd_kernel', 'og_gn_bwd_finalize_kernel',
         'og_affine_act_bwd_apply_kernel', 'og_gn_stats_kernel', 'og_gn_stats_split_kernel', 'og_gn_param_grads_kernel',
         'og_adagn_cond_fwd_kernel', 'og_adagn_cond_bwd_kernel']
    for w in want:
        assert any(w in n for n in names), (w, sorted(set(n for n in names if 'og_' in n)))
