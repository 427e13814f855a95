"""The fused residual-block node (ops._ResBlockFn: one autograd node for a whole VideoResidualBlock or
ImageResidualBlock without down-sampling) on every path it routes through, against a float64 restatement of the block.

The reference (`block_ref`) starts from x as bf16 and rounds to bf16 where the product does:
    a1 = bf16(act(GN1(x)))      h1 = bf16(conv1(a1) + b1)      a2 = bf16(act(GN2(h1)))
    y  = bf16(conv2(a2) + b2 + shortcut(x) + bres)
with GroupNorm statistics in float64, conv weights rounded to bf16, the padding of ops.ConvGeom (causal: kt - 1 frames
in front; symmetric: (kt - 1) // 2; space: (k - 1) // 2) and LeakyReLU's slope 0.01 (csrc/norm_act.cu). Its backward is
float64 autograd of that composition with every rounding passed straight through. The product's backward rounds d_a2,
d_h1, d_a1 and the shortcut's data gradient to bf16; the reference does not, and the end-to-end bounds below account
for it.

Two kinds of check:
- Staged, per element and tight. y.grad_fn.saved_tensors holds what the node saved (xi, a1, h1, a2, A1, B1, A2, B2, mr,
  ...), so every stage is checked against float64 computed from the kernel's own previous stage: the statistics (mr)
  against float64 statistics of the stage input; A, B against the kernel's mr; a1 / a2 against act(x A + B) from the
  kernel's A, B; h1 from a1 and y from a2 and xi by the convolution reference of conv_ref.py with its bound
  gam(n) sum|terms| (+ U |ref| for the bf16 rounding); y_sums against the float64 sums of the returned y; and, from the
  kernel's bf16 dy and the saved a2 / xi, dw2, dwres, db2 and dbres.
- End-to-end, for the gradients that depend on intermediates the node does not keep (dw1, db1, dgamma1/2, dbeta1/2,
  dx): against the rounded reference, per element within KE * U * (|ref| + rms(ref)), and in relative L2 below
  E2E_REL_L2. The per-element bound counts bf16 roundings of one ulp each, every one scaled by the rms of the tensor it
  lands in: the four of the backward, and a flip of the forward's a1, h1, a2 and y roundings, each reaching the
  gradient twice (through the value and through the GroupNorm statistics); 16 ulps in all.

Every case also asserts which path the IgemmPlan mirror says each forward GEMM takes, the exact list of C-ABI calls
(_lib.TIMING), and the same bits from two runs and from runs with the zero arena on and off.

The swapped-tile case is too large for a dense float64 forward on every voxel: its convolution stages are compared on
a sample of voxels gathered patch by patch, and its end-to-end gradients are not checked (its staged ones are). Its
tile box spans 128 x 2 x 1 voxels, so every voxel lies on a tile edge in H or T; the sample is a subset of those edges
(see sample_voxels), not all of them.
"""
import math
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from conv_ref import BF16, F32, F32T, F64T, SLACK, U, check, fwd_ref, gam, wgrad_ref
from test_gpu_conv_fwd_dgrad_paths import WS_FULL, IgemmPlan, num_sms

GPU = pytest.mark.gpu
DEV = 'cuda'
ONE = (1, 1, 1)
EPS = 1e-5
LEAKY = 0.01
ETANH = 2.0 ** -10.98       # tanh.approx.f32, PTX ISA: maximum relative error about 2^-11
TINY = 2.0 ** -100
KE = 16                     # end-to-end bound, in bf16 ulps of (|ref| + rms(ref)): see the module docstring
E2E_REL_L2 = 1e-2
ACT = {'none': 0, 'silu': 1, 'leaky': 2, 'relu': 3}
MARGINS = {}                # (case, quantity) -> worst err / bound seen, printed with -s


# ------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ------------------------------------------------------------------------------------------------------------------
def act_fn(pre, act):
    if act == 1:
        return pre * torch.sigmoid(pre)
    if act == 2:
        return torch.where(pre > 0, pre, LEAKY * pre)
    if act == 3:
        return pre.clamp_min(0)
    return pre


def act_grad(v, act):
    if act == 1:
        s = torch.sigmoid(v)
        return s * (1 + v * (1 - s))
    if act == 2:
        return torch.where(v > 0, torch.ones_like(v), torch.full_like(v, LEAKY))
    if act == 3:
        return (v > 0).to(v.dtype)
    return torch.ones_like(v)


class _ActAtOutput(torch.autograd.Function):
    """The activation with its derivative taken at its output instead of its input: a wiring mistake for the
    sensitivity tests."""

    @staticmethod
    def forward(ctx, pre, act):
        y = act_fn(pre, act)
        ctx.save_for_backward(y)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        return g * act_grad(y, ctx.act), None


def rnd(t):
    """bf16 rounding in the forward, identity in the backward."""
    return t + (t.to(BF16).to(t.dtype) - t).detach()


def gn_stats(x, G):
    """float64 (mean, var) per (sample, group) of x [N, T, H, W, C]: [N, G] each."""
    N, C = x.shape[0], x.shape[-1]
    xg = x.reshape(N, -1, G, C // G)
    mean = xg.mean((1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean((1, 3))
    return mean, var


def gn(x, G, gamma, beta, stats=None):
    N, C = x.shape[0], x.shape[-1]
    mean, var = gn_stats(x, G) if stats is None else stats
    xg = x.reshape(N, -1, G, C // G)
    xh = ((xg - mean[:, None, :, None]) / torch.sqrt(var[:, None, :, None] + EPS)).reshape(x.shape)
    return xh * gamma + beta


def block_ref(x, p, c, rounded=True, mut=()):
    """The block on x [N, T, H, W, C0] (float64 holding bf16 values); p: float64 parameters, conv weights as
    [cout, taps, cin] (bf16 values), the shortcut as [C1, C0]. `mut` names deliberate wiring mistakes (sensitivity
    tests only). Returns the stages {a1, h1, a2, y}."""
    r = rnd if rounded else (lambda t: t)
    act, G, k, pad, ext = ACT[c['act']], c['G'], c['k'], c['pad'], c['ext']
    act1 = (lambda v: _ActAtOutput.apply(v, act)) if 'act_grad_at_output' in mut else (lambda v: act_fn(v, act))
    s1 = None
    if 'stale_sums' in mut:
        s1 = gn_stats(p['x_before'], G)
    if 'other_sample_sums' in mut:
        s1 = tuple(t.roll(1, 0) for t in gn_stats(x, G))
    a1 = r(act1(gn(x, G, p['g1w'], p['g1b'], s1)))
    b1 = [] if p.get('b1') is None or 'no_conv1_bias' in mut else [p['b1']]
    h1 = r(fwd_ref(a1, p['w1'], k, ONE, pad, ext, biases=b1))
    a2 = r(act1(gn(h1, 1 if 'gn2_one_group' in mut else G, p['g2w'], p['g2b'])))
    xs = x.detach() if 'no_shortcut_dgrad' in mut else x
    wres = p['wres_shifted'] if 'shortcut_at_k_main_plus_64' in mut else p['wres']
    bs = [b for b in (p.get('b2'), p.get('bres')) if b is not None]
    y = r(fwd_ref(a2, p['w2'], k, ONE, pad, ext, x1=xs, w1=wres, biases=bs))
    return dict(a1=a1, h1=h1, a2=a2, y=y)


def torch_block(x5, p5, c):
    """The same block from torch modules in float64, without rounding: x5 NCDHW, p5 with 5-D conv weights."""
    act = {'none': nn.Identity(), 'silu': nn.SiLU(), 'leaky': nn.LeakyReLU(LEAKY), 'relu': nn.ReLU()}[c['act']]
    C0, C1, G = x5.shape[1], p5['w1'].shape[0], c['G']
    kt, kh, kw = c['k']
    pt, ph, pw = c['pad']

    def gnm(C, w, b):
        m = nn.GroupNorm(G, C, eps=EPS).double()
        with torch.no_grad():
            m.weight.copy_(w)
            m.bias.copy_(b)
        return m

    def conv(t, w, b):
        tp = F.pad(t, (pw, kw - 1 - pw, ph, kh - 1 - ph, pt, kt - 1 - pt))
        return F.conv3d(tp, w, b)
    h = conv(act(gnm(C0, p5['g1w'], p5['g1b'])(x5)), p5['w1'], p5['b1'])
    h = conv(act(gnm(C1, p5['g2w'], p5['g2b'])(h)), p5['w2'], p5['b2'])
    return h + F.conv3d(x5, p5['wres'], p5['bres'])


# ------------------------------------------------------------------------------------------------------------------
# the case table
# ------------------------------------------------------------------------------------------------------------------
def rc(G, C0, C1, k, causal, B, ext, act, sums, kernels, biases='all', image=False, large=False):
    """A node case. sums / kernels: the GroupNorm-sums path and (block_n, mn_major, wide, swap) of the two forward
    GEMMs as IgemmPlan derives them; biases: which of (b1, b2, bres) exist."""
    k = (k, k, k) if isinstance(k, int) else k
    pad = (k[0] - 1 if causal else (k[0] - 1) // 2, (k[1] - 1) // 2, (k[2] - 1) // 2)
    return dict(G=G, C0=C0, C1=C1, k=k, causal=causal, pad=pad, B=B, ext=ext, act=act, sums=sums, kernels=kernels,
                biases=biases, image=image, large=large)


K128, K256, WIDE, SWAP = (128, 0, False, False), (256, 0, True, False), (256, 0, True, False), (256, 0, True, True)
BIASES = {'all': 'b1 b2 bres', 'none': '', 'b1_bres': 'b1 bres', 'b2': 'b2'}

CASES = {
    # the shape of test_gpu_layers.py::test_video_residual_block: h1's sums from conv1's epilogue, y's from conv2's
    # split-K finish pass (55 k-blocks on 4 tiles split 6 ways)
    'golden_shape': rc(1, 64, 128, 3, False, 2, (4, 8, 8), 'silu', ('fused', 'finish'), (K128, K128)),
    # partial boxes in H and W, three samples with their own sums (both GEMMs split K on 9 tiles)
    'odd_extents': rc(1, 128, 128, 3, True, 3, (3, 6, 10), 'silu', ('finish', 'finish'), (K128, K128)),
    # G > 1: og_gn_stats for x and h1; C0 > C1, so the shortcut segment is wider than a conv2 tap
    'narrowing_stats': rc(4, 128, 64, 3, False, 2, (4, 8, 8), 'relu', (None, 'fused'), ((64, 0, False, False),) * 2),
    # ImageResidualBlock geometry: (1, 3, 3) kernels at T = 1, LeakyReLU
    'image_geometry': rc(8, 64, 64, (1, 3, 3), False, 2, (1, 16, 16), 'leaky', (None, 'fused'),
                         ((64, 0, False, False),) * 2, image=True),
    # one 4-sample box per tile: both GEMMs split K, their sums come out of the finish pass
    'splitk_finish': rc(1, 256, 256, 3, True, 1, (2, 4, 4), 'none', ('finish', 'finish'), (K128, K128)),
    # conv1 on the wide 128 x 256 tile with its fused sums
    'wide_tiles': rc(1, 64, 256, 3, True, 2, (4, 8, 8), 'silu', ('fused', 'finish'), (WIDE, K128)),
    # 163840 voxels >= 4 * 256 * SMs: swapped 256-voxel tiles for both GEMMs; sampled voxels
    'swapped_tiles': rc(1, 128, 128, 3, True, 2, (5, 128, 128), 'silu', ('fused', 'fused'), (SWAP, SWAP), large=True),
    # 1x1x1 main convolutions: one tap, the shortcut at k_main = C1
    'k1_main_convs': rc(2, 64, 128, 1, True, 2, (3, 5, 7), 'leaky', (None, 'fused'), (K128, K128)),
    # C / G = 8: the narrowest group the fused GroupNorm passes take
    'many_groups': rc(16, 128, 128, 3, False, 2, (2, 8, 8), 'relu', (None, 'finish'), (K128, K128)),
    # one box of 8 samples holds all 6 and K is not split: og_conv3d_fwd takes both GEMMs' sums from its own
    # og_gn_stats launch
    'stats_pass': rc(1, 128, 128, (1, 3, 3), False, 6, (1, 4, 4), 'silu', ('stats', 'stats'), (K128, K128)),
    **{f'biases_{b}': rc(1, 64, 128, 3, True, 2, (2, 8, 8), 'silu', ('fused', 'finish'), (K128, K128), biases=b)
       for b in BIASES},
}


def ws_bytes(c):
    B, V = c['B'], math.prod(c['ext'])
    return min(max(B * V * c['C1'] * 4, WS_FULL), 1 << 30)       # ops.StepScope.workspace for _workspace(B V C1 4)


def plans(c, sms):
    """IgemmPlan of conv1 (sums only when G = 1) and conv2 (+ the shortcut segment, always with sums)."""
    ws = ws_bytes(c)
    p1 = IgemmPlan(sms, False, c['C0'], c['k'], c['B'], c['ext'], c['C1'], ws_bytes=ws, sums=c['G'] == 1)
    p2 = IgemmPlan(sms, False, c['C1'], c['k'], c['B'], c['ext'], c['C1'], c1=c['C0'], ws_bytes=ws, sums=True)
    return p1, p2


def assert_paths(name, c, sms):
    p1, p2 = plans(c, sms)
    assert (p1.sums, p2.sums) == c['sums'], (name, sms, p1.describe(), p2.describe())
    assert (p1.kernel, p2.kernel) == c['kernels'], (name, sms, p1.describe(), p2.describe())
    assert not p1.refused and not p2.refused
    return p1, p2


def expected_calls(c, handed=False):
    """The node's C-ABI calls, forward then backward, for internal bf16 x and dy."""
    stats_x = [] if handed else ['og_gn_stats']
    stats_h1 = ['og_gn_stats'] if c['G'] > 1 else []
    fwd = stats_x + ['og_gn_act_fwd', 'og_conv3d_fwd'] + stats_h1 + ['og_gn_act_fwd', 'og_conv3d_fwd']
    bwd = ['og_conv3d_wgrad', 'og_conv3d_wgrad_bias', 'og_conv3d_dgrad', 'og_affine_act_bwd_reduce', 'og_gn_act_bwd',
           'og_conv3d_wgrad', 'og_conv3d_dgrad', 'og_affine_act_bwd_reduce', 'og_conv3d_dgrad', 'og_gn_act_bwd']
    return fwd, bwd


# ------------------------------------------------------------------------------------------------------------------
# operands (generated on the CPU, so that a CPU rehearsal sees the same data)
# ------------------------------------------------------------------------------------------------------------------
def make_params(c, seed):
    """fp32 parameters in the layouts the node takes: 5-D conv weights in channels_last_3d memory, [C] vectors.
    Conv1's bias carries a per-group offset and x per-sample / per-group scales, so that statistics taken over the
    wrong group or sample show."""
    g = torch.Generator().manual_seed(seed)
    C0, C1, G, k = c['C0'], c['C1'], c['G'], c['k']
    nt = math.prod(k)

    def rn(*s):
        return torch.randn(*s, generator=g)
    p = {'w1': rn(C1, C0, *k) / math.sqrt(C0 * nt), 'w2': rn(C1, C1, *k) / math.sqrt(C1 * nt),
         'wres': rn(C1, C0, 1, 1, 1) / math.sqrt(C0),
         'g1w': 1 + 0.25 * rn(C0), 'g1b': 0.25 * rn(C0), 'g2w': 1 + 0.25 * rn(C1), 'g2b': 0.25 * rn(C1),
         'b1': 0.3 * rn(C1) + 0.5 * (torch.arange(C1) // (C1 // G) % 3 - 1), 'b2': 0.3 * rn(C1), 'bres': 0.3 * rn(C1)}
    for key in ('w1', 'w2', 'wres'):
        p[key] = p[key].contiguous(memory_format=torch.channels_last_3d)
    for b in ('b1', 'b2', 'bres'):
        if b not in BIASES[c['biases']].split():
            p[b] = None
    return p


def make_x(c, seed, scale=1.0):
    """bf16 input [B, T, H, W, C0] (channels-last rows; the node's internal layout)."""
    g = torch.Generator().manual_seed(seed)
    B, C0, G = c['B'], c['C0'], c['G']
    n = torch.arange(B, dtype=F32T)[:, None]
    grp = torch.arange(C0)[None] // (C0 // G)
    sc = (1 + 0.5 * n + 0.25 * (grp % 3)) * scale
    off = 0.3 * (n - (grp % 3))
    x = torch.randn(B, *c['ext'], C0, generator=g) * sc[:, None, None, None] + off[:, None, None, None]
    return x.to(BF16)


def make_dy(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(c['B'], *c['ext'], c['C1'], generator=g).to(BF16)


def as_internal(rows):
    """[B, T, H, W, C] rows -> the logical (B, C, T, H, W) view the node takes."""
    return rows.permute(0, 4, 1, 2, 3)


def rows_of(t):
    """logical (B, C, T, H, W) -> [B, T, H, W, C]."""
    return t.permute(0, 2, 3, 4, 1)


def ref_params(p, dev, x=None):
    """float64 reference parameters: conv weights rounded to bf16, as [cout, taps, cin]."""
    def w(t):
        cout, cin = t.shape[0], t.shape[1]
        return t.detach().to(BF16).double().permute(0, 2, 3, 4, 1).reshape(cout, -1, cin).to(dev)
    q = {'w1': w(p['w1']), 'w2': w(p['w2']), 'wres': w(p['wres'])[:, 0, :]}
    for key in ('g1w', 'g1b', 'g2w', 'g2b', 'b1', 'b2', 'bres'):
        q[key] = None if p[key] is None else p[key].detach().double().to(dev)
    return q


# ------------------------------------------------------------------------------------------------------------------
# bounds
# ------------------------------------------------------------------------------------------------------------------
def stats_expect(x, G, partial=None):
    """(mean, rstd) float64 of x [N, ..., C] and their bounds, for fp64 sums of fp32 partials of at most `partial`
    terms (default: the whole group, which bounds every sums path; the large case passes one swapped tile's outputs,
    the longest fp32 partial of its epilogue sums, og_gn_stats's per-thread partials being shorter)."""
    N, C = x.shape[0], x.shape[-1]
    xg = x.reshape(N, -1, G, C // G)
    cnt = xg.shape[1] * xg.shape[3]
    mean, var = gn_stats(x, G)
    rstd = 1 / torch.sqrt(var + EPS)
    e = gam(min(cnt, partial or cnt) + 64)
    emean = e * xg.abs().sum((1, 3)) / cnt
    evar = e * (xg * xg).sum((1, 3)) / cnt + (2 * mean.abs() + emean) * emean
    q = evar / (var + EPS)
    assert float(q.max()) < 0.5, 'statistics too imprecise for the linearised rstd bound'
    rel = q / (1 - q) + F32
    return (mean, SLACK * (emean + F32 * mean.abs()) + TINY), (rstd, SLACK * rel * rstd + TINY)


def coef_expect(mr, gamma, beta, C):
    """A = rstd gamma and B = beta - mean rstd gamma from the kernel's own fp32 (mean, rstd): a few fp32 roundings."""
    N, G = mr.shape[0], mr.shape[1]
    mu = mr[..., 0].double().repeat_interleave(C // G, 1)
    rs = mr[..., 1].double().repeat_interleave(C // G, 1)
    A = rs * gamma
    m = mu * A
    Bc = beta - m
    return (A, SLACK * F32 * A.abs() + TINY), (Bc, SLACK * F32 * (2 * m.abs() + Bc.abs()) + TINY)


def act_expect(x, A, Bc, act):
    """act(x A + B) from the kernel's own coefficients, then the bf16 rounding: x [N, ..., C], A / B [N, C]. The fma
    rounds once; SiLU is h (1 + tanh(h)) at h = pre / 2 (1.1-Lipschitz, plus the tanh.approx error)."""
    sh = (x.shape[0],) + (1,) * (x.dim() - 2) + (x.shape[-1],)
    pre = x * A.view(sh) + Bc.view(sh)
    y = act_fn(pre, act)
    if act == 1:
        e = 1.1 * F32 * pre.abs() + 0.5 * pre.abs() * ETANH * torch.tanh(pre / 2).abs() + 3 * F32 * y.abs()
    else:
        e = F32 * (pre.abs() + y.abs())
    return y, SLACK * e + U * y.abs() + TINY


def conv_expect(x, w, c, plan, x1=None, w1=None, biases=()):
    """One convolution stage against conv_ref.fwd_ref: gam(k-products + split slabs + biases) sum|terms|, then one
    bf16 rounding."""
    ref = fwd_ref(x, w, c['k'], ONE, c['pad'], c['ext'], x1=x1, w1=w1, biases=biases)
    mag = fwd_ref(x.abs(), w.abs(), c['k'], ONE, c['pad'], c['ext'], x1=None if x1 is None else x1.abs(),
                  w1=None if w1 is None else w1.abs(), biases=[b.abs() for b in biases])
    n = plan.num_kb * 64 + plan.splits + 3
    return ref, (1 + U) * gam(n) * SLACK * mag + U * ref.abs() + TINY


def sums_expect(y, partial=None):
    """float64 (sum, sum of squares) per sample of the bf16 y, and the bound of fp32 partials of at most `partial`
    terms (default: the sample)."""
    yf = y.double().reshape(y.shape[0], -1)
    want = torch.stack([yf.sum(1), (yf * yf).sum(1)], 1)[:, None]
    mag = torch.stack([yf.abs().sum(1), (yf * yf).sum(1)], 1)[:, None]
    return want, gam(min(yf.shape[1], partial or yf.shape[1]) + 64) * SLACK * mag + TINY


def wgrad_expect(x, dy, k, pad, sms):
    """dW [cout, taps, cin] of the bf16 dy and x; n = voxels + the stream-K segments a tile may be cut into + 1."""
    ref = wgrad_ref(x, dy, k, ONE, pad)
    mag = wgrad_ref(x.abs(), dy.abs(), k, ONE, pad)
    n = x.shape[0] * math.prod(x.shape[1:4]) + 2 * sms + 1
    return ref, gam(n) * SLACK * mag + TINY


def e2e_bound(ref):
    ref = ref.double()
    rms = ref.pow(2).mean().sqrt()
    return KE * U * (ref.abs() + rms) + TINY


def check_m(case, name, got, ref, tol):
    """conv_ref.check, recording the worst err / bound."""
    got, ref = got.double().to(ref.device), ref.double()
    tol = torch.as_tensor(tol, dtype=F64T, device=ref.device).expand_as(ref)
    ratio = float(((got - ref).abs() / tol).nan_to_num(float('inf')).max()) if ref.numel() else 0.0
    MARGINS[(case, name)] = max(MARGINS.get((case, name), 0.0), ratio)
    check(f'{case} {name}', got, ref, tol)


def check_e2e(case, name, got, ref):
    check_m(case, name, got, ref, e2e_bound(ref))
    r = rel_l2(got, ref)
    MARGINS[(case, name + ' rel_l2')] = max(MARGINS.get((case, name + ' rel_l2'), 0.0), r / E2E_REL_L2)
    assert r < E2E_REL_L2, f'{case} {name}: relative L2 {r:.3g}'


def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten().to(a.device)
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------------------------
# running the node
# ------------------------------------------------------------------------------------------------------------------
def node_inputs(c, seed, dev=DEV):
    from open_genie_b200 import ops
    p = make_params(c, seed)
    geom1 = ops.ConvGeom(c['C0'], c['C1'], c['k'], causal=c['causal'])
    geom2 = ops.ConvGeom(c['C1'], c['C1'], c['k'], causal=c['causal'])
    pd = {k: None if v is None else v.to(dev) for k, v in p.items()}
    packed1 = torch.zeros((c['C1'], geom1.kpad), dtype=BF16, device=dev)
    packed2 = torch.zeros((c['C1'], geom2.kpad + c['C0']), dtype=BF16, device=dev)
    ops.pack_weight(pd['w1'], packed1, 0)
    ops.pack_weight(pd['w2'], packed2, 0)
    ops.pack_weight(pd['wres'], packed2, geom2.kpad)
    return dict(p=pd, geom1=geom1, geom2=geom2, packed1=packed1, packed2=packed2,
                x=make_x(c, seed + 1).to(dev), dy=make_dy(c, seed + 2).to(dev))


PARAMS = ('g1w', 'g1b', 'w1', 'b1', 'g2w', 'g2b', 'w2', 'b2', 'wres', 'bres')


def run_node(c, d, x=None, dy=None, sums=None, grad=True, frozen=(), x_grad=True):
    """One forward (+ backward of dy) of ops.residual_block. Returns the outputs, the saved stages, the gradients
    and the C-ABI calls of the forward and the backward."""
    from open_genie_b200 import _lib, ops
    x = as_internal(d['x']) if x is None else x
    dy = as_internal(d['dy']) if dy is None else dy
    leaves = {k: None if v is None else v.detach().clone().requires_grad_(grad and k not in frozen)
              for k, v in d['p'].items()}
    xg = x.detach().clone(memory_format=torch.preserve_format).requires_grad_(grad and x_grad)
    out = {}
    _lib.TIMING = []
    try:
        y, ys = ops.residual_block(xg, sums, *(leaves[k] for k in PARAMS), d['packed1'], d['packed2'], d['geom1'],
                                   d['geom2'], c['G'], EPS, act=c['act'])
        out['fwd_calls'] = [t[0] for t in _lib.TIMING]
        out['y'], out['y_sums'] = y.detach().clone(), ys.clone()
        if y.grad_fn is not None:
            out['saved'] = [t.detach().clone() for t in y.grad_fn.saved_tensors[:9]]
        if grad:
            _lib.TIMING = []
            torch.autograd.backward(y, dy)
            out['bwd_calls'] = [t[0] for t in _lib.TIMING]
        torch.cuda.synchronize()
    finally:
        _lib.TIMING = None
    if grad:
        out['grads'] = {k: None if v is None or v.grad is None else v.grad.detach().clone() for k, v in leaves.items()}
        out['grads']['x'] = None if xg.grad is None else xg.grad.detach().clone()
    return out


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == BF16 else torch.int32 if t.dtype == F32T else torch.int64)


def assert_same_bits(what, a, b):
    for key in ('y', 'y_sums'):
        assert torch.equal(bits(a[key]), bits(b[key])), f'{what}: {key} differs'
    for k, g in a.get('grads', {}).items():
        h = b['grads'][k]
        assert (g is None) == (h is None), (what, k)
        if g is not None:
            assert torch.equal(bits(g), bits(h)), f'{what}: gradient of {k} differs'


# ------------------------------------------------------------------------------------------------------------------
# staged and end-to-end checks
# ------------------------------------------------------------------------------------------------------------------
def sample_voxels(c, plan, n_random=2048, seed=0):
    """[M, 4] (n, t, h, w) voxel indices of the large case. The box spans one frame and two rows, so every voxel is on
    a tile edge in T and H and checking all tile-edge voxels would mean checking them all; this is a subset: every
    voxel on a W face of a box, whole rows at the first, middle and last box row, the first and last voxel of each
    sample, and random voxels."""
    B, (T, H, W) = c['B'], c['ext']
    bw, bh = plan.box[0], plan.box[1]
    grids = []
    n, t, h = torch.meshgrid(torch.arange(B), torch.arange(T), torch.arange(H), indexing='ij')
    for w0 in sorted({w for b in range(0, W, bw) for w in (b, min(b + bw, W) - 1)}):
        grids.append(torch.stack([n.flatten(), t.flatten(), h.flatten(), torch.full_like(n.flatten(), w0)], 1))
    rows = sorted({r for b in (0, (H // bh // 2) * bh, (H // bh - 1) * bh) for r in range(b, min(b + bh, H))})
    n, t, h, w = torch.meshgrid(torch.arange(B), torch.arange(T), torch.tensor(rows), torch.arange(W), indexing='ij')
    grids.append(torch.stack([n.flatten(), t.flatten(), h.flatten(), w.flatten()], 1))
    ends = [(b, 0, 0, 0) for b in range(B)] + [(b, T - 1, H - 1, W - 1) for b in range(B)]
    grids.append(torch.tensor(ends))
    g = torch.Generator().manual_seed(seed)
    grids.append(torch.stack([torch.randint(0, e, (n_random,), generator=g) for e in (B, T, H, W)], 1))
    return torch.unique(torch.cat(grids), dim=0)


def fwd_at(x, w, c, idx, x1=None, w1=None, biases=(), chunk=2048):
    """fwd_ref at the voxels idx only, by gathering each voxel's input patch: (ref, sum |terms|) [M, cout]."""
    k, pad = c['k'], c['pad']
    T, H, W = c['ext']
    taps = [(a, b, e) for a in range(k[0]) for b in range(k[1]) for e in range(k[2])]
    refs, mags = [], []
    for i0 in range(0, idx.shape[0], chunk):
        ix = idx[i0:i0 + chunk].to(x.device)
        cols = []
        for (a, b, e) in taps:
            pt, ph, pw = ix[:, 1] + a - pad[0], ix[:, 2] + b - pad[1], ix[:, 3] + e - pad[2]
            ok = (pt >= 0) & (pt < T) & (ph >= 0) & (ph < H) & (pw >= 0) & (pw < W)
            v = x[ix[:, 0], pt.clamp(0, T - 1), ph.clamp(0, H - 1), pw.clamp(0, W - 1)]
            cols.append(v * ok[:, None].to(v.dtype))
        patch = torch.stack(cols, 1)                                   # [m, taps, cin]
        r = torch.einsum('mtc,otc->mo', patch, w)
        m = torch.einsum('mtc,otc->mo', patch.abs(), w.abs())
        if x1 is not None:
            v1 = x1[ix[:, 0], ix[:, 1], ix[:, 2], ix[:, 3]]
            r, m = r + v1 @ w1.T, m + v1.abs() @ w1.abs().T
        for bb in biases:
            r, m = r + bb, m + bb.abs()
        refs.append(r)
        mags.append(m)
    return torch.cat(refs), torch.cat(mags)


def at(t, idx):
    ix = idx.to(t.device)
    return t[ix[:, 0], ix[:, 1], ix[:, 2], ix[:, 3]]


def staged_checks(name, c, d, out, sms):
    """Each saved stage against float64 computed from the kernel's previous stage."""
    p1, p2 = plans(c, sms)
    q = ref_params(d['p'], DEV)
    G, act = c['G'], ACT[c['act']]
    xi, a1, h1, a2, A1, B1, A2, B2, mr = out['saved']
    xi, a1, h1, a2 = (rows_of(t).double() for t in (xi, a1, h1, a2))
    y = rows_of(out['y']).double()
    assert torch.equal(xi, d['x'].double()), f'{name}: the saved input is not x'
    partial = 256 * max(c['C0'], c['C1']) if c['large'] else None
    for stage, (src, gw, gb, A, Bc, m, dst) in {'gn1': (xi, q['g1w'], q['g1b'], A1, B1, mr[0], a1),
                                                'gn2': (h1, q['g2w'], q['g2b'], A2, B2, mr[1], a2)}.items():
        (mean, emean), (rstd, erstd) = stats_expect(src, G, partial)
        check_m(name, f'{stage} mean', m[..., 0], mean, emean)
        check_m(name, f'{stage} rstd', m[..., 1], rstd, erstd)
        (Ar, eA), (Br, eB) = coef_expect(m, gw, gb, src.shape[-1])
        check_m(name, f'{stage} A', A, Ar, eA)
        check_m(name, f'{stage} B', Bc, Br, eB)
        yr, ey = act_expect(src, A.double(), Bc.double(), act)
        check_m(name, f'{stage} out', dst, yr, ey)
    b1 = [] if q['b1'] is None else [q['b1']]
    bs = [b for b in (q['b2'], q['bres']) if b is not None]
    n1, n2 = p1.num_kb * 64 + p1.splits + 3, p2.num_kb * 64 + p2.splits + 3
    if c['large']:
        idx = sample_voxels(c, p2)
        r, mag = fwd_at(a1, q['w1'], c, idx, biases=b1)
        check_m(name, 'h1 (sampled)', at(h1, idx), r, (1 + U) * gam(n1) * SLACK * mag + U * r.abs() + TINY)
        r, mag = fwd_at(a2, q['w2'], c, idx, x1=xi, w1=q['wres'], biases=bs)
        check_m(name, 'y (sampled)', at(y, idx), r, (1 + U) * gam(n2) * SLACK * mag + U * r.abs() + TINY)
    else:
        check_m(name, 'h1', h1, *conv_expect(a1, q['w1'], c, p1, biases=b1))
        check_m(name, 'y', y, *conv_expect(a2, q['w2'], c, p2, x1=xi, w1=q['wres'], biases=bs))
    check_m(name, 'y_sums', out['y_sums'], *sums_expect(y, partial))
    if 'grads' not in out:
        return
    gr = out['grads']
    dyb = d['dy'].double()
    C0, C1 = c['C0'], c['C1']
    check_m(name, 'dw2', gr['w2'].permute(0, 2, 3, 4, 1).reshape(C1, -1, C1), *wgrad_expect(a2, dyb, c['k'], c['pad'],
                                                                                             sms))
    r, e = wgrad_expect(xi, dyb, ONE, (0, 0, 0), sms)
    check_m(name, 'dwres', gr['wres'].reshape(C1, C0), r[:, 0], e[:, 0])
    db = dyb.reshape(-1, C1).sum(0)
    edb = gam(dyb.numel() // C1 + 2 * sms + 1) * SLACK * dyb.abs().reshape(-1, C1).sum(0) + TINY
    for key in ('b2', 'bres'):
        if q[key] is None:
            assert gr[key] is None, f'{name}: a gradient for the missing {key}'
        else:
            check_m(name, f'd{key}', gr[key], db, edb)
    if q['b2'] is not None and q['bres'] is not None:
        assert torch.equal(gr['b2'], gr['bres']), f'{name}: db2 and dbres differ'
    if q['b1'] is None:
        assert gr['b1'] is None, f'{name}: a gradient for the missing b1'


def e2e_reference(c, d, dev=None, mut=()):
    """float64 autograd of block_ref for dy: (the stages, the gradients by parameter name and 'x')."""
    dev = dev or DEV
    q = ref_params(d['p'], dev)
    leaves = {k: None if v is None else v.clone().requires_grad_(True) for k, v in q.items()}
    x = d['x'].double().to(dev).requires_grad_(True)
    if 'stale_sums' in mut or 'shortcut_at_k_main_plus_64' in mut:
        leaves.update({k: d[k] for k in ('x_before', 'wres_shifted') if k in d})
    st = block_ref(x, leaves, c, mut=mut)
    st['y'].backward(d['dy'].double().to(dev))
    grads = {k: None if v is None or not isinstance(v, torch.Tensor) or v.grad is None else v.grad
             for k, v in leaves.items()}
    grads['x'] = x.grad
    return st, grads


E2E = ('g1w', 'g1b', 'w1', 'b1', 'g2w', 'g2b', 'x')


def e2e_checks(name, c, d, out):
    _, gref = e2e_reference(c, d)
    gr = out['grads']
    for k in E2E:
        if gref.get(k) is None:
            assert gr.get(k) is None, (name, k)
            continue
        got = gr[k]
        if k == 'w1':
            got = got.permute(0, 2, 3, 4, 1).reshape(gref[k].shape)
        elif k == 'x':
            got = rows_of(got)
        check_e2e(name, f'd{k}', got, gref[k])


def print_margins(name):
    for (case, q), v in sorted(MARGINS.items()):
        if case == name:
            print(f'margin {case} {q}: {v:.3g}')


# ------------------------------------------------------------------------------------------------------------------
# GPU: the case table
# ------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize('name', list(CASES))
def test_node_case(name):
    from open_genie_b200 import ops
    c = CASES[name]
    sms = num_sms()
    p1, p2 = assert_paths(name, c, sms)
    print(f'{name}: conv1 {p1.describe()}; conv2 {p2.describe()}')
    d = node_inputs(c, zlib.crc32(name.encode()))
    out = run_node(c, d)
    fwd, bwd = expected_calls(c)
    assert out['fwd_calls'] == fwd, (name, out['fwd_calls'])
    assert out['bwd_calls'] == bwd, (name, out['bwd_calls'])
    staged_checks(name, c, d, out, sms)
    if not c['large']:
        e2e_checks(name, c, d, out)
    assert_same_bits(f'{name}: a second run', out, run_node(c, d))
    prev = ops.current_arena()
    ops.enable_zero_arena(True)
    try:
        ops.mark_step()
        on = run_node(c, d)
    finally:
        ops.enable_zero_arena(prev is not None)
    assert_same_bits(f'{name}: zero arena on', out, on)
    print_margins(name)


# ------------------------------------------------------------------------------------------------------------------
# GPU: paths through the Python wrapper
# ------------------------------------------------------------------------------------------------------------------
LAYOUT_CASE = CASES['narrowing_stats']


@GPU
def test_layouts_frozen_parameters_and_no_grad():
    """x and dy as internal bf16 or NCDHW fp32 (the same values), x without a gradient, a frozen parameter subset
    and a no_grad forward all give the bits of the internal bf16 run."""
    from open_genie_b200 import ops
    c = LAYOUT_CASE
    d = node_inputs(c, 11)
    base = run_node(c, d)
    x32 = ops.to_reference(as_internal(d['x']))
    dy32 = ops.to_reference(as_internal(d['dy']))
    assert x32.is_contiguous() and x32.dtype == F32T
    for what, kw in (('x NCDHW fp32', dict(x=x32)), ('dy NCDHW fp32', dict(dy=dy32)),
                     ('both NCDHW fp32', dict(x=x32, dy=dy32))):
        out = run_node(c, d, **kw)
        assert out['fwd_calls'][0] == ('og_ncdhw_f32_to_ndhwc' if 'x' in kw else 'og_gn_stats'), out['fwd_calls']
        gx = out['grads'].pop('x')
        assert_same_bits(what, dict(base, grads={k: v for k, v in base['grads'].items() if k != 'x'}), out)
        assert torch.equal(gx.float(), base['grads']['x'].float()), f'{what}: dx differs'
    out = run_node(c, d, x_grad=False)
    assert out['grads']['x'] is None
    assert_same_bits('x without a gradient', dict(base, grads={k: v for k, v in base['grads'].items() if k != 'x'}),
                     dict(out, grads={k: v for k, v in out['grads'].items() if k != 'x'}))
    frozen = ('g1w', 'w2', 'b1', 'bres')
    out = run_node(c, d, frozen=frozen)
    for k in frozen:
        assert out['grads'][k] is None, k
    assert_same_bits('frozen parameters', dict(base, grads={k: v for k, v in base['grads'].items() if k not in frozen}),
                     dict(out, grads={k: v for k, v in out['grads'].items() if k not in frozen}))
    with torch.no_grad():
        ng = run_node(c, d, grad=False)
    assert 'saved' not in ng
    assert ng['fwd_calls'] == expected_calls(c)[0]
    assert_same_bits('no_grad forward', dict(base, grads={}), ng)


def _blocks(G1, seed=3):
    from open_genie_b200.module.video import VideoResidualBlock
    torch.manual_seed(seed)
    return VideoResidualBlock(64, 128, num_groups=G1).to(DEV), VideoResidualBlock(128).to(DEV)


def _calls(fn):
    from open_genie_b200 import _lib
    _lib.TIMING = []
    try:
        r = fn()
        torch.cuda.synchronize()
        return r, [t[0] for t in _lib.TIMING]
    finally:
        _lib.TIMING = None


def _consumer(b2, h, dy):
    """b2's output and its parameter gradients for upstream dy, and the calls its forward made."""
    b2.zero_grad(set_to_none=True)
    y, calls = _calls(lambda: b2(h))
    if torch.is_grad_enabled():
        y.backward(dy)
    grads = {k: p.grad.clone() for k, p in b2.named_parameters() if p.grad is not None}
    return y.detach().clone(), grads, calls


def _sums_match_stats(h):
    """Whether the handed-over sums of h equal og_gn_stats's bit for bit; returns (equal, handed, recomputed)."""
    from open_genie_b200 import _lib, ops
    handed = h._og_gn_sums[0].clone()
    B, C, T, H, W = h.shape
    fresh = torch.zeros((B, 1, 2), dtype=F64T, device=DEV)
    _lib.call('og_gn_stats', h.data_ptr(), B, T * H * W, C, 1, fresh.data_ptr(), ops._stream())
    torch.cuda.synchronize()
    return torch.equal(handed, fresh), handed, fresh


def bf16_ulp(t):
    """One bf16 ulp of each element of t (float64; 0 where t is 0): 2^(e - 8) for |t| in [2^(e-1), 2^e)."""
    t = t.double()
    _, e = torch.frexp(t)
    return torch.where(t == 0, torch.zeros_like(t), torch.ldexp(torch.ones_like(t), e - 8))


def _assert_consumer_match(tag, a, b, exact):
    """Consumer results a against b: the same bits, or (exact=False) every element of the output and of every
    gradient within one bf16 ulp of b's."""
    ya, ga = a[0], a[1]
    yb, gb = b[0], b[1]
    assert set(ga) == set(gb), tag
    if exact:
        assert torch.equal(bits(ya), bits(yb)), f'{tag}: output differs'
        for k in ga:
            assert torch.equal(bits(ga[k]), bits(gb[k])), f'{tag}: gradient of {k} differs'
        return
    check(f'{tag} y', ya, yb.double(), bf16_ulp(yb))
    for k in ga:
        check(f'{tag} d{k}', ga[k], gb[k].double(), bf16_ulp(gb[k]))


@GPU
@pytest.mark.parametrize('G1', [1, 8])
def test_handed_over_sums(G1):
    """A producer with G1 groups hands G = 1 sums of its output to a G = 1 consumer; the consumer uses them (no
    og_gn_stats) and matches itself run on a copy, which recomputes them with og_gn_stats. The epilogue's sums are
    fp32 partials per tile combined in fp64, og_gn_stats's fp32 partials per thread: the same sums to within the bound
    of sums_expect but not the same bits, so the consumer is held to one bf16 ulp per element, not to equal bits."""
    torch.manual_seed(5)
    b1, b2 = _blocks(G1)
    x = torch.randn((2, 64, 3, 8, 8), device=DEV)
    dy = torch.randn((2, 128, 3, 8, 8), device=DEV).to(BF16)
    h = b1(x.requires_grad_(True))
    sums = h._og_gn_sums[0]
    assert sums.shape == (2, 1, 2)
    want, tol = sums_expect(rows_of(h.detach()))
    check('handed-over sums', sums, want, tol)
    exact, handed, fresh = _sums_match_stats(h)
    assert not exact, 'the epilogue sums now equal og_gn_stats bit for bit: hold the consumer to equal bits'
    check('og_gn_stats sums', fresh, want, tol)
    used = _consumer(b2, h, dy)
    assert 'og_gn_stats' not in used[2], used[2]
    fresh_run = _consumer(b2, h.detach().clone(), dy)
    assert fresh_run[2].count('og_gn_stats') == 1, fresh_run[2]
    _assert_consumer_match(f'G1 = {G1}', used, fresh_run, False)
    same = torch.equal(bits(used[0]), bits(fresh_run[0])) and all(torch.equal(used[1][k], fresh_run[1][k])
                                                                  for k in used[1])
    print(f'handed-over sums, G1 = {G1}: consumer output and gradients bit-equal to the recomputed run: {same}')


@GPU
def test_inference_mode_chain():
    """Under torch.inference_mode() (tensors without a version counter) no sums are handed over: the consumer
    recomputes them, and the chain gives the bits of a no_grad chain whose consumer runs on a copy."""
    torch.manual_seed(8)
    b1, b2 = _blocks(1)
    x = torch.randn((2, 64, 3, 8, 8), device=DEV)
    with torch.inference_mode():
        h, c1 = _calls(lambda: b1(x))
        assert h.is_inference() and not hasattr(h, '_og_gn_sums')
        y, c2 = _calls(lambda: b2(h))
    assert c1.count('og_gn_stats') == 1 and c2.count('og_gn_stats') == 1, (c1, c2)
    with torch.no_grad():
        hn = b1(x)
        yn = b2(hn.clone())
    assert torch.equal(bits(h), bits(hn)) and torch.equal(bits(y), bits(yn))


@GPU
@pytest.mark.parametrize('grad', [False, True])
def test_sums_are_not_reused_after_an_in_place_edit(grad):
    """An in-place edit of a block's output keeps the Python attribute; the next block must recompute its
    statistics and give what it gives on a copy. In grad mode the producer is frozen: autograd refuses an in-place edit
    of an output that has a grad_fn (a view made inside a custom Function), so a frozen block feeding a trained one is
    where an edited output reaches a block whose backward runs."""
    torch.manual_seed(6)
    b1, b2 = _blocks(1)
    b1.requires_grad_(False)
    x = torch.randn((2, 64, 3, 8, 8), device=DEV)
    dy = torch.randn((2, 128, 3, 8, 8), device=DEV).to(BF16)
    with torch.set_grad_enabled(grad):
        h = b1(x)
        assert h.grad_fn is None
        h.mul_(3.0)
        bad = _consumer(b2, h, dy)
        good = _consumer(b2, h.detach().clone(), dy)
    assert bad[2].count('og_gn_stats') == 1, f'the edited tensor\'s stale sums were reused: {bad[2]}'
    _assert_consumer_match('after an in-place edit', bad, good, True)


@GPU
def test_sums_are_not_reused_across_an_arena_step():
    """With the zero arena on, the handed-over sums live in the step's arena; after mark_step() and one allocation they
    have been zeroed, so a block fed an output kept across the step must recompute them."""
    from open_genie_b200 import ops
    torch.manual_seed(7)
    b1, b2 = _blocks(1)
    x = torch.randn((2, 64, 3, 8, 8), device=DEV, requires_grad=True)
    dy = torch.randn((2, 128, 3, 8, 8), device=DEV).to(BF16)
    prev = ops.current_arena()
    ops.enable_zero_arena(True)
    try:
        ops.mark_step()
        h = b1(x)
        assert ops.current_arena().locate(h._og_gn_sums[0]) is not None
        ops.mark_step()
        ops._zeros(16, F32T, DEV)
        kept = _consumer(b2, h, dy)
        fresh = _consumer(b2, h.detach().clone(), dy)
    finally:
        ops.enable_zero_arena(prev is not None)
    assert kept[2].count('og_gn_stats') == 1, f'sums from an earlier arena step were reused: {kept[2]}'
    _assert_consumer_match('across an arena step', kept, fresh, True)


MODULE_CASES = [(causal, G, act) for causal in (True, False) for G in (1, 2, 8) for act in ('silu', 'leaky', 'relu')]


def _module_ref_case(m, x, image):
    """The node case and float64 parameters of module m, from its state_dict."""
    sd = {k: v.detach().float().cpu() for k, v in m.state_dict().items()}
    if image:
        pre = {'g1': 'main.0', 'c1': 'main.2', 'g2': 'main.3', 'c2': 'main.5', 'res': 'res'}
        k = (1,) + tuple(sd['main.2.weight'].shape[2:])
        causal, act, G = False, 'leaky', m.main[0].num_groups
    else:
        cv = '.conv3d' if m.use_causal else ''
        pre = {'g1': 'main.0', 'c1': f'main.2{cv}', 'g2': 'main.4', 'c2': f'main.6{cv}', 'res': f'res.1{cv}'}
        k = tuple(sd[pre['c1'] + '.weight'].shape[2:])
        causal, act, G = m.use_causal, m.act_fn, m.main[0].num_groups
    w5 = lambda t: t if t.dim() == 5 else t.unsqueeze(2)
    p = {'g1w': sd['main.0.weight'], 'g1b': sd['main.0.bias'], 'g2w': sd[pre['g2'] + '.weight'],
         'g2b': sd[pre['g2'] + '.bias'], 'w1': w5(sd[pre['c1'] + '.weight']), 'b1': sd[pre['c1'] + '.bias'],
         'w2': w5(sd[pre['c2'] + '.weight']), 'b2': sd[pre['c2'] + '.bias'], 'wres': w5(sd[pre['res'] + '.weight']),
         'bres': sd[pre['res'] + '.bias']}
    B, C0, T, H, W = x.shape
    c = rc(G, C0, p['w1'].shape[0], k, causal, B, (T, H, W), act, None, None)
    return c, p


def _module_check(tag, m, x, dy, image=False):
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    y.backward(dy)
    c, p = _module_ref_case(m, x, image)
    d = {'p': p, 'x': rows_of(x).to(BF16), 'dy': rows_of(dy)}
    st, gref = e2e_reference(c, d)
    check_e2e(tag, 'y', rows_of(y.detach()), st['y'].detach())
    check_e2e(tag, 'dx', rows_of(xg.grad), gref['x'])
    names = {'g1w': m.main[0].weight, 'w1': m.main[2].weight if image else
             (m.main[2].conv3d.weight if m.use_causal else m.main[2].weight)}
    check_e2e(tag, 'dg1w', names['g1w'].grad, gref['g1w'])
    check_e2e(tag, 'dw1', names['w1'].grad.permute(0, 2, 3, 4, 1).reshape(gref['w1'].shape), gref['w1'])
    return y


@GPU
@pytest.mark.parametrize('causal,G,act', MODULE_CASES)
def test_video_block_routing(causal, G, act):
    """VideoResidualBlock runs the fused node (only it sets _og_gn_sums) and matches the reference built from its
    state_dict."""
    from open_genie_b200.module.video import VideoResidualBlock
    torch.manual_seed(G * 10 + int(causal))
    m = VideoResidualBlock(64, 128, num_groups=G, use_causal=causal, act_fn=act).to(DEV)
    x = torch.randn((2, 64, 3, 6, 6), device=DEV).to(BF16).float()
    dy = torch.randn((2, 128, 3, 6, 6), device=DEV).to(BF16).float()
    y = _module_check(f'video causal={causal} G={G} {act}', m, x, dy)
    assert hasattr(y, '_og_gn_sums') and type(y.grad_fn).__name__ == '_ResBlockFnBackward'


@GPU
@pytest.mark.parametrize('G', [1, 8, 16])
def test_image_block_routing(G):
    """ImageResidualBlock on the fused node (C / G a multiple of 8) and on the layer-by-layer path (64 / 16 = 4)."""
    from open_genie_b200.module.image import ImageResidualBlock
    torch.manual_seed(40 + G)
    m = ImageResidualBlock(64, 128, num_groups=G).to(DEV)
    x = torch.randn((2, 64, 1, 8, 8), device=DEV).to(BF16).float()
    dy = torch.randn((2, 128, 1, 8, 8), device=DEV).to(BF16).float()
    y = _module_check(f'image G={G}', m, x, dy, image=True)
    fused = type(y.grad_fn).__name__ == '_ResBlockFnBackward'
    assert fused == (G != 16), type(y.grad_fn).__name__


@GPU
@pytest.mark.parametrize('kind,G', [('image', 16), ('image', 1), ('video', 16), ('video', 1)])
def test_fused_adamw_step_updates_the_shortcut(kind, G):
    """After one FusedAdamW step a block computes what a fresh block loaded from its state_dict computes, bit for bit:
    every bf16 copy of a weight, the shortcut's included, follows the fp32 parameter."""
    from open_genie_b200.module.image import ImageResidualBlock
    from open_genie_b200.module.video import VideoResidualBlock
    from open_genie_b200.optim import FusedAdamW
    make = (lambda: ImageResidualBlock(64, 128, num_groups=G)) if kind == 'image' else \
        (lambda: VideoResidualBlock(64, 128, num_groups=G))
    torch.manual_seed(50 + G)
    m = make().to(DEV)
    x = torch.randn((2, 64, 1 if kind == 'image' else 3, 8, 8), device=DEV)
    m(x).float().square().mean().backward()
    FusedAdamW(m.parameters(), lr=0.05).step()
    m.zero_grad(set_to_none=True)
    fresh = make().to(DEV)
    fresh.load_state_dict(m.state_dict())
    with torch.no_grad():
        a, b = m(x), fresh(x)
    torch.cuda.synchronize()
    assert torch.equal(bits(a), bits(b)), f'{kind} G={G}: the stepped block and its state_dict copy differ'


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference, the bounds and the plan
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('act', list(ACT))
@pytest.mark.parametrize('causal', [True, False])
def test_reference_matches_torch_modules(act, causal):
    c = rc(2, 8, 16, 3, causal, 2, (3, 4, 5), act, None, None)
    p = make_params(c, 1)
    q = {k: v.double() for k, v in p.items()}
    x5 = torch.randn(2, 8, 3, 4, 5, dtype=F64T)
    want = torch_block(x5, q, c)
    qr = {'w1': q['w1'].permute(0, 2, 3, 4, 1).reshape(16, 27, 8), 'w2': q['w2'].permute(0, 2, 3, 4, 1).reshape(16, 27, 16),
          'wres': q['wres'][:, :, 0, 0, 0]}
    qr.update({k: q[k] for k in ('g1w', 'g1b', 'g2w', 'g2b', 'b1', 'b2', 'bres')})
    got = block_ref(rows_of(x5), qr, c, rounded=False)['y']
    err = float((rows_of(want) - got.detach()).abs().max())
    assert err <= 1e-12 * float(want.abs().max()), err
    # and the backward of the two compositions
    xa, xb = x5.clone().requires_grad_(True), x5.clone().requires_grad_(True)
    g = torch.randn_like(want)
    torch_block(xa, q, c).backward(g)
    block_ref(rows_of(xb), qr, c, rounded=False)['y'].backward(rows_of(g))
    assert float((xa.grad - xb.grad).abs().max()) <= 1e-12 * float(xa.grad.abs().max())


@pytest.mark.parametrize('sms', [114, 132])
def test_cases_take_their_paths(sms):
    for name, c in CASES.items():
        assert_paths(name, c, sms)
    seen = {s for c in CASES.values() for s in c['sums']}
    assert seen == {None, 'fused', 'finish', 'stats'}
    kernels = {kk for c in CASES.values() for kk in c['kernels']}
    assert {WIDE, SWAP} <= kernels


def test_expected_calls_pin_og_gn_stats():
    for c in CASES.values():
        fwd, _ = expected_calls(c)
        assert fwd.count('og_gn_stats') == 1 + (c['G'] > 1) and fwd.count('og_conv3d_fwd') == 2
        assert expected_calls(c, handed=True)[0].count('og_gn_stats') == (c['G'] > 1)


def _cpu_case(name):
    c = CASES[name]
    d = node_inputs_cpu(c, zlib.crc32(name.encode()))
    return c, d


def node_inputs_cpu(c, seed):
    return dict(p=make_params(c, seed), x=make_x(c, seed + 1), dy=make_dy(c, seed + 2))


def _staged_from_ref(c, d, st):
    """The staged bounds evaluated on the reference's own stages (as if the kernel had computed them exactly)."""
    q = ref_params(d['p'], 'cpu')
    G, act = c['G'], ACT[c['act']]
    x = d['x'].double()
    out = {}
    for stage, (src, gw, gb, dst) in {'gn1': (x, q['g1w'], q['g1b'], st['a1']),
                                      'gn2': (st['h1'], q['g2w'], q['g2b'], st['a2'])}.items():
        (mean, emean), (rstd, erstd) = stats_expect(src.detach(), G)
        mr = torch.stack([mean, rstd], -1).float()
        (A, _), (Bc, _) = coef_expect(mr, gw, gb, src.shape[-1])
        A, Bc = A.float().double(), Bc.float().double()
        out[stage] = act_expect(src.detach(), A, Bc, act)
        out[stage + ' stats'] = ((mean, emean), (rstd, erstd))
    plan1, plan2 = plans(c, 132)
    b1 = [] if q['b1'] is None else [q['b1']]
    bs = [b for b in (q['b2'], q['bres']) if b is not None]
    out['h1'] = conv_expect(st['a1'].detach(), q['w1'], c, plan1, biases=b1)
    out['y'] = conv_expect(st['a2'].detach(), q['w2'], c, plan2, x1=x, w1=q['wres'], biases=bs)
    return out


def _rejects(what, got, ref, tol):
    with pytest.raises(AssertionError):
        check(what, got, ref, tol)


@pytest.mark.parametrize('name', ['golden_shape', 'narrowing_stats'])
def test_bounds_reject_wiring_mistakes(name):
    c, d = _cpu_case(name)
    d['x_before'] = d['x'].double()
    xe = (d['x'].double() * 3).to(BF16)
    q = ref_params(d['p'], 'cpu')
    ws = torch.zeros_like(q['wres'])
    ws[:, :c['C0'] - 64] = q['wres'][:, 64:]            # columns k_main + 64 on: the rest of the shortcut, then zeros
    d['wres_shifted'] = ws
    st, gref = e2e_reference(c, d, 'cpu')
    stages = _staged_from_ref(c, d, st)
    # the reference passes its own bounds
    check('a1', st['a1'], *stages['gn1'])
    check('h1', st['h1'], *stages['h1'])
    check('a2', st['a2'], *stages['gn2'])
    check('y', st['y'], *stages['y'])

    def e2e(mut):
        return e2e_reference(c, d, 'cpu', mut=mut)
    # backward wiring, end to end
    _, g = e2e(('no_shortcut_dgrad',))
    _rejects('the shortcut data gradient dropped', g['x'], gref['x'], e2e_bound(gref['x']))
    _rejects('db1 := db2', gref['b2'], gref['b1'], e2e_bound(gref['b1']))
    _rejects('dgamma and dbeta swapped', gref['g1b'], gref['g1w'], e2e_bound(gref['g1w']))
    _rejects('dgamma and dbeta swapped', gref['g2b'], gref['g2w'], e2e_bound(gref['g2w']))
    if c['act'] == 'silu':
        _, g = e2e(('act_grad_at_output',))
        _rejects('the activation derivative at its output', g['x'], gref['x'], e2e_bound(gref['x']))
        _rejects('the activation derivative at its output', g['w1'], gref['w1'], e2e_bound(gref['w1']))
    # forward wiring, per stage
    m, _ = e2e(('no_conv1_bias',))
    _rejects('conv1 bias omitted', m['h1'], *stages['h1'])
    m, _ = e2e(('shortcut_at_k_main_plus_64',))
    _rejects('the shortcut read from k_main + 64', m['y'], *stages['y'])
    if c['G'] > 1:
        m, _ = e2e(('gn2_one_group',))
        _rejects('GN2 statistics with G = 1', m['a2'], *stages['gn2'])
    (mean, emean), (rstd, erstd) = stages['gn1 stats']
    _rejects("another sample's mean", mean.roll(1, 0), mean, emean)
    _rejects("another sample's rstd", rstd.roll(1, 0), rstd, erstd)
    m, _ = e2e(('other_sample_sums',))
    _rejects("another sample's sums", m['a1'], st['a1'], e2e_bound(st['a1']))
    # stale sums: x edited (x 3) after its statistics were taken
    de = dict(d, x=xe)
    ste, _ = e2e_reference(c, de, 'cpu')
    (mean3, emean3), (rstd3, erstd3) = stats_expect(xe.double(), c['G'])
    _rejects('stale mean', mean, mean3, emean3)
    _rejects('stale rstd', rstd, rstd3, erstd3)
    m, _ = e2e_reference(c, de, 'cpu', mut=('stale_sums',))
    _rejects('stale sums', m['a1'], ste['a1'], e2e_bound(ste['a1']))


def test_sample_covers_the_w_faces_and_sample_ends():
    c = CASES['swapped_tiles']
    _, p2 = plans(c, 132)
    idx = sample_voxels(c, p2)
    B, (T, H, W) = c['B'], c['ext']
    bw = p2.box[0]
    assert p2.box[:3] == (128, 2, 1)
    have = {tuple(v) for v in idx.tolist()}
    for n in range(B):
        for t in range(T):
            for h in range(H):
                for w in (0, bw - 1):
                    assert (n, t, h, w) in have
        assert (n, 0, 0, 0) in have and (n, T - 1, H - 1, W - 1) in have


def test_patch_gather_equals_the_dense_reference():
    """fwd_at (the large case's sampled convolution) gives fwd_ref's values and magnitudes at the sampled voxels."""
    c = rc(1, 8, 8, 3, True, 2, (3, 5, 6), 'silu', None, None)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 5, 6, 8, generator=g, dtype=F64T)
    x1 = torch.randn(2, 3, 5, 6, 8, generator=g, dtype=F64T)
    w = torch.randn(8, 27, 8, generator=g, dtype=F64T)
    w1 = torch.randn(8, 8, generator=g, dtype=F64T)
    b = torch.randn(8, generator=g, dtype=F64T)
    idx = torch.unique(torch.stack([torch.randint(0, e, (64,), generator=g) for e in (2, 3, 5, 6)], 1), dim=0)
    idx = torch.cat([idx, torch.tensor([[0, 0, 0, 0], [1, 2, 4, 5]])])
    r, m = fwd_at(x, w, c, idx, x1=x1, w1=w1, biases=[b], chunk=7)
    dense = fwd_ref(x, w, c['k'], ONE, c['pad'], c['ext'], x1=x1, w1=w1, biases=[b])
    dmag = fwd_ref(x.abs(), w.abs(), c['k'], ONE, c['pad'], c['ext'], x1=x1.abs(), w1=w1.abs(), biases=[b.abs()])
    assert float((r - at(dense, idx)).abs().max()) <= 1e-12 * float(dense.abs().max())
    assert float((m - at(dmag, idx)).abs().max()) <= 1e-12 * float(dmag.abs().max())


def test_image_block_without_fusable_shortcut_channels_is_refused():
    """A 1x1 shortcut runs as extra K columns of the last convolution, on either image-block path: channel counts that
    are not multiples of 64 raise NotImplementedError before any kernel (this runs without a device)."""
    from open_genie_b200.module.image import ImageResidualBlock
    for cin, cout, G in ((32, 32, 16), (32, 64, 1), (64, 96, 1)):
        m = ImageResidualBlock(cin, cout, num_groups=G)
        with pytest.raises(NotImplementedError, match='multiples of 64'):
            m(torch.zeros(1, cin, 1, 4, 4))
