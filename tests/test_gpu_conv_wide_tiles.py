"""The 128 x 256 tiles of og_conv_igemm_kernel (both consumer warpgroups on one item, m64n256k16 each) through the C ABI:
forward with K-major weights and data gradient with MN-major weights, the bias pair with the fused 1x1x1 shortcut
segment, residual, GroupNorm sums, a partial last N tile, partial voxel boxes, and one item per CTA / one item more than
the grid; and the swapped 256-voxel x 128-channel tiles (forward, MN-major data gradient, the tokenizer's 3-channel
tail, shortcut segment, GroupNorm sums, partial boxes). Outputs are pre-filled with NaN and compared element by element with torch in fp32 (TF32 off) on the same
bf16 operands; two calls must give the same bits. A profiler test pins each convolution shape class of the tokenizer
step to the kernel variant launch_igemm promises for it."""
import re
import zlib

import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda'
BF16_HALF_ULP = 2.0 ** -8    # largest relative rounding error of a bf16 output


def _gen(name):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(f'conv_wide_{name}'.encode()))


def _rand(g, shape, scale=1.0):
    return ((torch.rand(shape, generator=g, device=DEV) * 2 - 1) * scale).to(torch.bfloat16)


def _no_tf32(fn):
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _conv_ref(x, w, k):
    """fp32 causal convolution (front time padding k - 1, symmetric space padding) of channels-last x with packed
    w [cout][tap][cin]; returns NCDHW."""
    cout, cin = w.shape[0], x.shape[-1]
    wt = w.float().reshape(cout, k, k, k, cin).permute(0, 4, 1, 2, 3)
    p = (k - 1) // 2
    return F.conv3d(F.pad(x.float().permute(0, 4, 1, 2, 3), (p, p, p, p, k - 1, 0)), wt)


def _fwd(x, w, k, cout, bias0=None, bias1=None, x1=None, residual=None, sums=False, ws_bytes=0):
    """og_conv3d_fwd into a NaN-filled bf16 output: (out, GroupNorm sums or None). Without workspace no launch splits."""
    from open_genie_b200 import _lib
    N, T, H, W, cin = x.shape
    c1 = x1.shape[-1] if x1 is not None else 0
    out = torch.full((N, T, H, W, cout), float('nan'), dtype=torch.bfloat16, device=DEV)
    gs = torch.zeros((N, 2), dtype=torch.float64, device=DEV) if sums else None
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    pad = (k - 1) // 2
    _lib.call('og_conv3d_fwd', x.data_ptr(), cin, k, k, k, k - 1, pad, pad, p(x1), c1, w.data_ptr(), w.shape[1], p(bias0),
              p(bias1), p(residual), out.data_ptr(), 0, N, T, H, W, cout, ws.data_ptr() if ws_bytes else None, ws_bytes,
              p(gs), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out, gs


def _dgrad(dy, w, k, cin, ws_bytes=0):
    from open_genie_b200 import _lib
    N, T, H, W, cout = dy.shape
    dx = torch.full((N, T, H, W, cin), float('nan'), dtype=torch.bfloat16, device=DEV)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    pad = (k - 1) // 2
    _lib.call('og_conv3d_dgrad', dy.data_ptr(), cout, w.shape[0], w.data_ptr(), w.shape[1], 0, k, k, k, k - 1, pad, pad,
              dx.data_ptr(), 0, N, T, H, W, cin, ws.data_ptr() if ws_bytes else None, ws_bytes,
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dx


def _dgrad_ref(dy, w, k, in_shape):
    x = torch.zeros(in_shape, device=DEV, requires_grad=True)

    def run():
        _conv_ref(x, w, k).backward(dy.float().permute(0, 4, 1, 2, 3))
        return x.grad
    return _no_tf32(run)


def _check_fwd(name, out, ref, sums, out2):
    assert_close(out, ref, 2e-3 + BF16_HALF_ULP, 1e-3 * ref.abs().max().item(), f'{name} forward')
    if sums is not None:
        N = out.shape[0]
        y = out.double().reshape(N, -1)
        assert torch.all((sums[:, 0] - y.sum(1)).abs() <= 1e-4 * y.abs().sum(1)), f'{name}: GroupNorm sum'
        assert torch.all((sums[:, 1] - (y * y).sum(1)).abs() <= 1e-4 * (y * y).sum(1)), f'{name}: GroupNorm sum of squares'
    assert torch.equal(out, out2), f'{name}: two calls differ'


def _check_dgrad(name, dy, w, k, cin):
    dx = _dgrad(dy, w, k, cin)
    ref = _dgrad_ref(dy, w, k, dy.shape[:4] + (cin,))
    assert_close(dx, ref, 2e-3 + BF16_HALF_ULP, 1e-3 * ref.abs().max().item(), f'{name} data gradient')
    assert torch.equal(dx, _dgrad(dy, w, k, cin)), f'{name}: two data-gradient calls differ'


@pytest.mark.parametrize('cout', [256, 320, 512])
def test_forward_bias_groupnorm(cout):
    """256 -> cout, 3x3x3, bias and GroupNorm sums; 320 leaves one 64-column chunk in the last N tile."""
    Ci, k, N = 256, 3, 2
    g = _gen(f'fwd_{cout}')
    x = _rand(g, (N, 4, 8, 16, Ci))
    w = _rand(g, (cout, k ** 3 * Ci), 0.05)
    bias = torch.rand(cout, generator=g, device=DEV) * 2 - 1
    out, sums = _fwd(x, w, k, cout, bias0=bias, sums=True)
    out2, _ = _fwd(x, w, k, cout, bias0=bias, sums=True)
    ref = _no_tf32(lambda: _conv_ref(x, w, k) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd(f'{cout} channels', out, ref, sums, out2)


@pytest.mark.parametrize('cin', [256, 320])
def test_mn_major_dgrad(cin):
    """Data gradient with MN-major weights: 4 panels of 64 input channels per stage; 320 = a partial last N tile."""
    Co, k, N = 128, 3, 2
    g = _gen(f'dgrad_{cin}')
    dy = _rand(g, (N, 4, 8, 16, Co))
    w = _rand(g, (Co, k ** 3 * cin), 0.1)
    _check_dgrad(f'cin {cin}', dy, w, k, cin)


def test_fused_shortcut_bias_pair_groupnorm():
    """3x3x3 over 128 channels + the 1x1x1 shortcut over 128 channels into 256 outputs, bias0 + bias1, GroupNorm sums."""
    C0, C1, Co, k, N = 128, 128, 256, 3, 2
    g = _gen('fused')
    x0 = _rand(g, (N, 4, 16, 16, C0))
    x1 = _rand(g, (N, 4, 16, 16, C1))
    w = _rand(g, (Co, k ** 3 * C0 + C1), 0.1)
    b0 = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    b1 = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    out, sums = _fwd(x0, w, k, Co, bias0=b0, bias1=b1, x1=x1, sums=True)
    out2, _ = _fwd(x0, w, k, Co, bias0=b0, bias1=b1, x1=x1, sums=True)

    def ref():
        y = _conv_ref(x0, w[:, :k ** 3 * C0], k)
        y = y + torch.einsum('nthwc,oc->nothw', x1.float(), w[:, k ** 3 * C0:].float())
        return (y + (b0 + b1).view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd('fused shortcut', out, _no_tf32(ref), sums, out2)


def test_residual_partial_boxes():
    """out = conv + bias + residual on a 3 x 12 x 20 grid: the voxel boxes overhang along t, h and w."""
    Ci, Co, k, N = 64, 256, 3, 2
    g = _gen('residual')
    x = _rand(g, (N, 3, 12, 20, Ci))
    w = _rand(g, (Co, k ** 3 * Ci), 0.1)
    res = _rand(g, (N, 3, 12, 20, Co))
    bias = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    out, _ = _fwd(x, w, k, Co, bias0=bias, residual=res)
    out2, _ = _fwd(x, w, k, Co, bias0=bias, residual=res)
    ref = _no_tf32(lambda: _conv_ref(x, w, k) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1) + res.float()
    _check_fwd('residual', out, ref, None, out2)


def test_dgrad_partial_boxes():
    """Data gradient on a 3 x 10 x 12 grid: the voxel boxes overhang along w and h."""
    Ci, Co, k, N = 256, 64, 3, 2
    g = _gen('dgrad_partial')
    dy = _rand(g, (N, 3, 10, 12, Co))
    w = _rand(g, (Co, k ** 3 * Ci), 0.1)
    _check_dgrad('partial boxes', dy, w, k, Ci)


@pytest.mark.parametrize('items', ['one_per_cta', 'grid_plus_one'])
def test_item_counts(items):
    """128 x 1 x 1 voxel tiles, one per W row, 256 output channels: `rows` items of 27 k-blocks each, a count that does
    not divide the stage ring."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = {'one_per_cta': sms // 2, 'grid_plus_one': sms + 1}[items]
    C, k = 256, 3
    g = _gen(items)
    x = _rand(g, (1, 1, rows, 128, 64))
    dy = _rand(g, (1, 1, rows, 128, 64))
    w = _rand(g, (C, k ** 3 * 64), 0.2)
    bias = torch.rand(C, generator=g, device=DEV) * 2 - 1
    out, sums = _fwd(x, w, k, C, bias0=bias, sums=True)
    out2, _ = _fwd(x, w, k, C, bias0=bias, sums=True)
    ref = _no_tf32(lambda: _conv_ref(x, w, k) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd(items, out, ref, sums, out2)
    wd = _rand(g, (64, k ** 3 * C), 0.2)    # a 256 -> 64 convolution: its data gradient has 256 outputs
    _check_dgrad(items, dy, wd, k, C)


# Swapped tiles (256 voxels x 128 channels) need >= 4 tiles per SM: 2 x 10 x 120 x 60 voxels = 600 tiles of 64 x 4 x 1,
# the last w box of each row overhanging by 4, and a tile count that is no multiple of the grid.
SWAP_GRID = (2, 10, 120, 60)


@pytest.mark.parametrize('case', ['bias_groupnorm', 'residual', 'shortcut_bias_pair'])
def test_swapped_forward(case):
    """128 output channels with the operands swapped: the weights are the K-major A operand, the activation box B.
    (With a residual the same shape runs the ping-pong kernel: checked here on the same grid all the same.)"""
    N, T, H, W = SWAP_GRID
    C0, C1, Co, k = 64, (64 if case == 'shortcut_bias_pair' else 0), 128, 3
    g = _gen(f'swap_fwd_{case}')
    x0 = _rand(g, (N, T, H, W, C0))
    x1 = _rand(g, (N, T, H, W, C1)) if C1 else None
    w = _rand(g, (Co, k ** 3 * C0 + C1), 0.1)
    b0 = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    b1 = torch.rand(Co, generator=g, device=DEV) * 2 - 1 if C1 else None
    res = _rand(g, (N, T, H, W, Co)) if case == 'residual' else None
    sums = case != 'residual'
    out, gs = _fwd(x0, w, k, Co, bias0=b0, bias1=b1, x1=x1, residual=res, sums=sums)
    out2, _ = _fwd(x0, w, k, Co, bias0=b0, bias1=b1, x1=x1, residual=res, sums=sums)

    def ref():
        y = _conv_ref(x0, w[:, :k ** 3 * C0], k) + b0.view(1, -1, 1, 1, 1)
        if C1:
            y = y + torch.einsum('nthwc,oc->nothw', x1.float(), w[:, k ** 3 * C0:].float()) + b1.view(1, -1, 1, 1, 1)
        y = y.permute(0, 2, 3, 4, 1)
        return y + res.float() if res is not None else y
    _check_fwd(f'swapped {case}', out, _no_tf32(ref), gs, out2)


@pytest.mark.parametrize('cout', [128, 3])
def test_swapped_dgrad(cout):
    """Data gradient into 128 channels with the operands swapped: the weights are an MN-major A operand (A-transpose
    bit); cout = 3 is the tokenizer's tail, whose dy is zero-padded to 64 channels with 3 rows of weights."""
    N, T, H, W = SWAP_GRID
    Ci, k = 128, 3
    cpad = (cout + 63) // 64 * 64
    g = _gen(f'swap_dgrad_{cout}')
    dy = _rand(g, (N, T, H, W, cpad))
    if cpad != cout:
        dy[..., cout:] = 0
    w = _rand(g, (cout, k ** 3 * Ci), 0.1)
    from open_genie_b200 import _lib
    dx = torch.full((N, T, H, W, Ci), float('nan'), dtype=torch.bfloat16, device=DEV)

    def call():
        _lib.call('og_conv3d_dgrad', dy.data_ptr(), cpad, cout, w.data_ptr(), w.shape[1], 0, k, k, k, k - 1, 1, 1,
                  dx.data_ptr(), 0, N, T, H, W, Ci, None, 0, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return dx.clone()
    got = call()
    ref = _dgrad_ref(dy[..., :cout], w, k, (N, T, H, W, Ci))
    assert_close(got, ref, 2e-3 + BF16_HALF_ULP, 1e-3 * ref.abs().max().item(), f'swapped data gradient {cout}')
    assert torch.equal(got, call()), f'swapped data gradient {cout}: two calls differ'


# Shape classes of the tokenizer step (B = 8) and the og_conv_igemm_kernel<BN, MN-major, wide, swapped> each one
# launches. (kind, cin, cout, (T, H, W), shortcut channels, with GroupNorm sums) -> (BN, wide, swapped)
STEP_CLASSES = [
    (('fwd', 128, 128, (16, 64, 64), 0, True), (256, True, True)),
    (('fwd', 128, 128, (16, 64, 64), 256, True), (256, True, True)),
    (('fwd', 256, 128, (16, 64, 64), 0, True), (256, True, True)),
    (('fwd', 128, 256, (16, 32, 32), 0, True), (256, True, False)),
    (('fwd', 256, 256, (16, 32, 32), 128, True), (256, True, False)),
    (('fwd', 256, 256, (16, 32, 32), 0, True), (256, True, False)),
    (('fwd', 256, 1024, (16, 32, 32), 0, False), (256, True, False)),
    (('fwd', 256, 256, (8, 16, 16), 0, True), (256, True, False)),
    (('fwd', 256, 2048, (8, 16, 16), 0, False), (256, True, False)),
    (('fwd', 512, 256, (8, 16, 16), 0, True), (256, True, False)),
    (('fwd', 512, 4096, (4, 8, 8), 0, False), (256, True, False)),
    (('fwd', 512, 512, (4, 8, 8), 0, True), (128, False, False)),      # split-K
    (('dgrad', 128, 128, (16, 64, 64), 0, False), (256, True, True)),
    (('dgrad', 256, 128, (16, 64, 64), 0, False), (256, True, False)),
    (('dgrad', 256, 256, (16, 32, 32), 0, False), (256, True, False)),
    (('dgrad', 256, 1024, (16, 32, 32), 0, False), (256, True, False)),
    (('dgrad', 256, 256, (8, 16, 16), 0, False), (256, True, False)),
    (('dgrad', 256, 2048, (8, 16, 16), 0, False), (128, False, False)),   # measured slower on the wide tile
    (('dgrad', 512, 256, (8, 16, 16), 0, False), (128, False, False)),    # measured slower on the wide tile
    (('dgrad', 512, 512, (4, 8, 8), 0, False), (128, False, False)),   # split-K
]


def test_step_classes_dispatch():
    """Each shape class of the step, called as the step calls it (24 MiB of split-K workspace), launches the promised
    og_conv_igemm_kernel instantiation."""
    from torch.profiler import ProfilerActivity, profile
    B, k, ws_bytes = 8, 3, 24 << 20
    g = _gen('dispatch')
    for (kind, cin, cout, (T, H, W), sc, gn), (bn, wide, swap) in STEP_CLASSES:
        if kind == 'fwd':
            x = _rand(g, (B, T, H, W, cin))
            x1 = _rand(g, (B, T, H, W, sc)) if sc else None
            w = _rand(g, (cout, k ** 3 * cin + sc), 0.05)
            bias = torch.zeros(cout, device=DEV)
            call = lambda: _fwd(x, w, k, cout, bias0=bias, x1=x1, sums=gn, ws_bytes=ws_bytes)   # noqa: E731
        else:
            dy = _rand(g, (B, T, H, W, cout))
            w = _rand(g, (cout, k ** 3 * cin), 0.05)
            call = lambda: _dgrad(dy, w, k, cin, ws_bytes=ws_bytes)   # noqa: E731
        call()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        names = [e.name for e in prof.events() if 'og_conv_igemm_kernel' in e.name]
        got = {m.groups() for m in (re.search(r'og_conv_igemm_kernel<(\d+), (\d), (true|false), (true|false)>', n) for n in names) if m}
        want = {(str(bn), '1' if kind == 'dgrad' else '0', 'true' if wide else 'false', 'true' if swap else 'false')}
        assert got == want, f'{kind} {cin}->{cout} @{T}x{H}x{W}: launched {sorted(got)}, expected {sorted(want)}'
        del call
        torch.cuda.empty_cache()
