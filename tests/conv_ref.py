"""The float64 "convolution by taps" reference and the comparisons shared by the convolution path tests
(test_gpu_conv_wgrad_strided_paths.py, test_gpu_conv_fwd_dgrad_paths.py).

Rounding model, as in test_gpu_attention_paths.py: U is the unit roundoff of bf16, F32 one fp32 ulp per addition
(tensor-core sums may truncate), gam(n) the relative error of an n-term sum in any order."""
import itertools

import pytest
import torch
import torch.nn.functional as F

from helpers import Guarded

DEV = 'cuda'
BF16, F32T, F64T = torch.bfloat16, torch.float32, torch.float64

U = 2.0 ** -8
F32 = 2.0 ** -23
SLACK = 1.02
EXACT_LIMIT = 2 ** 22       # sum of |terms| per element for the exact checks


def gam(n):
    return n * F32


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------------------
# geometry and the float64 reference
# ------------------------------------------------------------------------------------------------------------------
def _taps(k):
    return list(itertools.product(range(k[0]), range(k[1]), range(k[2])))


def _positions(o, s, tap, pad, mut):
    """Input position of output o along one dimension for one tap."""
    return o * s + tap - pad + (1 if 'stride_off' in mut else 0)


def _mutate(k, pad, mut):
    taps = _taps(k)
    used = [tuple(kk - 1 - a for kk, a in zip(k, t)) for t in taps] if 'mirror' in mut else taps
    if 'causal_sym' in mut:
        pad = ((k[0] - 1) // 2, pad[1], pad[2])
    return taps, used, pad


def shift(x, tap, s, pad, out, mut=()):
    """x[n, o*s + tap - pad] over the output grid `out`, zero where that is outside x: one tap's operand."""
    y = x
    for d in range(3):
        n_in = x.shape[1 + d]
        pos = _positions(torch.arange(out[d], device=x.device), s[d], tap[d], pad[d], mut)
        ok = (pos >= 0) & (pos < n_in)
        y = y.index_select(1 + d, pos.clamp(0, n_in - 1))
        shape = [1] * 5
        shape[1 + d] = -1
        y = y * ok.view(shape).to(y.dtype)
    return y


def fwd_ref(x, w, k, s, pad, out, mut=(), x1=None, w1=None, biases=(), residual=None):
    """y[n, o, co] = sum_tap shift(x)[n, o] . w[co, tap]: x [N,T,H,W,cin], w [cout, ntaps, cin] -> [N, *out, cout].
    Optionally + x1 . w1^T (the second, 1x1x1 K segment: x1 [N, *out, c1], w1 [cout, c1]), + each bias [cout] and
    + residual [N, *out, cout]."""
    taps, used, pad = _mutate(k, pad, mut)
    y = 0
    for i, t in enumerate(used):
        y = y + shift(x, t, s, pad, out, mut) @ w[:, i, :].T
    if x1 is not None:
        y = y + x1 @ w1.T
    for b in biases:
        y = y + b
    if residual is not None:
        y = y + residual
    return y


def wgrad_ref(x, dy, k, s, pad, mut=()):
    """dW[co, tap, ci] = dY^T . shift(x): dy [N, *out, cout] -> [cout, ntaps, cin]."""
    taps, used, pad = _mutate(k, pad, mut)
    out = tuple(dy.shape[1:4])
    d2 = dy.reshape(-1, dy.shape[-1]).T
    return torch.stack([d2 @ shift(x, t, s, pad, out, mut).reshape(-1, x.shape[-1]) for t in used], 1)


def dgrad_ref(dy, w, k, s, pad, ext, mut=(), w_rows=None):
    """dx = sum_tap unshift(dY . w[:, tap]): dy [N, *out, cout], w [cout, ntaps, cin] -> [N, *ext, cin]. With w_rows,
    only the first w_rows rows of w and channels of dy take part (the rest of dy is zero padding)."""
    if w_rows is not None:
        dy, w = dy[..., :w_rows], w[:w_rows]
    taps, used, pad = _mutate(k, pad, mut)
    N, out, cin = dy.shape[0], tuple(dy.shape[1:4]), w.shape[2]
    T, H, W = ext
    dx = torch.zeros((N, T * H * W, cin), dtype=dy.dtype, device=dy.device)
    for i, t in enumerate(used):
        g = (dy.reshape(-1, dy.shape[-1]) @ w[:, i, :]).view(N, -1, cin)
        pos = [_positions(torch.arange(out[d], device=dy.device), s[d], t[d], pad[d], mut) for d in range(3)]
        ok = [(p >= 0) & (p < e) for p, e in zip(pos, ext)]
        lin = (pos[0][:, None, None] * H + pos[1][None, :, None]) * W + pos[2][None, None, :]
        m = (ok[0][:, None, None] & ok[1][None, :, None] & ok[2][None, None, :]).flatten()
        dx.index_add_(1, lin.flatten()[m], g[:, m])
    return dx.view(N, T, H, W, cin)


def torch_ref(op, x, w, dy, k, s, pad, ext):
    """The same three products from F.conv3d / torch.nn.grad on an explicitly padded input (causal time padding is
    one-sided, so it cannot be expressed as conv3d's symmetric padding)."""
    N, T, H, W, cin = x.shape
    cout = w.shape[0]
    out = dy.shape[1:4]
    back = [max(0, (o - 1) * ss + kk - p - e) for o, ss, kk, p, e in zip(out, s, k, pad, ext)]
    xp = F.pad(x.permute(0, 4, 1, 2, 3), (pad[2], back[2], pad[1], back[1], pad[0], back[0]))
    w5 = w.view(cout, *k, cin).permute(0, 4, 1, 2, 3)
    dy5 = dy.permute(0, 4, 1, 2, 3)
    if op == 'fwd':
        return F.conv3d(xp, w5, stride=s)[:, :, :out[0], :out[1], :out[2]].permute(0, 2, 3, 4, 1)
    # the padded input is cropped to what the strided windows reach, so that torch sees no partial window
    reach = [(o - 1) * ss + kk for o, ss, kk in zip(out, s, k)]
    xp = xp[:, :, :reach[0], :reach[1], :reach[2]]
    if op == 'wgrad':
        g = torch.nn.grad.conv3d_weight(xp, w5.shape, dy5, stride=s)
        return g.permute(0, 2, 3, 4, 1).reshape(cout, -1, cin)
    gx = torch.nn.grad.conv3d_input(xp.shape, w5, dy5, stride=s)
    gx = F.pad(gx, (0, max(0, W + pad[2] - reach[2]), 0, max(0, H + pad[1] - reach[1]), 0,
                    max(0, T + pad[0] - reach[0])))
    return gx[:, :, pad[0]:pad[0] + T, pad[1]:pad[1] + H, pad[2]:pad[2] + W].permute(0, 2, 3, 4, 1)


def voxel_box(vox, T, H, W):
    """choose_voxel_box (csrc/og_host.cu): widest-first powers of two over (W, H, T), the rest over samples."""
    def p2(v):
        p = 1
        while p < v:
            p *= 2
        return p
    w = min(p2(W), vox)
    rem = vox // w
    h = min(p2(H), rem)
    rem //= h
    t = min(p2(T), rem)
    rem //= t
    return w, h, t, min(rem, 256)


# ------------------------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------------------------
def check(name, got, ref, tol):
    """|got - ref| <= tol element by element (float64); a NaN or an unwritten (NaN-filled) element fails."""
    got, ref, tol = got.double(), ref.double(), torch.as_tensor(tol, dtype=F64T, device=ref.device)
    err = (got - ref).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        tolf = tol.expand_as(ref).flatten()
        raise AssertionError(f'{name}: {int(bad.sum())}/{bad.numel()} outside the bound; first at flat {i}: got '
                             f'{got.flatten()[i].item():.9g} ref {ref.flatten()[i].item():.9g} bound '
                             f'{tolf[i].item():.3g}')


def check_exact(name, got, ref):
    check(name, got, ref, 0.0)


def rejects(fn):
    with pytest.raises(AssertionError):
        fn()


def nan_bits(t):
    ity, bits = Guarded.BITS[t.dtype]
    return bool((t.contiguous().view(ity) == bits).all())


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def operand(shape, seed, kind, device=DEV, dtype=BF16, lo=-3, hi=3):
    """'int': integers in [lo, hi]; 'real': random signs, magnitudes 2^U(-10, 10) (no subnormals), rounded to dtype."""
    g = gen(seed, device)
    if kind == 'int':
        return torch.randint(lo, hi + 1, shape, generator=g, device=device).to(dtype)
    mag = torch.exp2(torch.rand(shape, generator=g, device=device, dtype=F64T) * 20 - 10)
    sign = torch.randint(0, 2, shape, generator=g, device=device) * 2 - 1
    return (mag * sign).to(dtype)
