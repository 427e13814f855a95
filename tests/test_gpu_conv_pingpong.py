"""The convolution forward and data gradient through the C ABI, on the launches where the two consumer warpgroups of
og_conv_igemm_kernel meet their edge cases: a CTA with one item (the second consumer idles), one item more than the
grid and an odd number of items per CTA (the consumers step over each other's k-blocks of the shared stage ring),
split items with different k-block counts, and every epilogue path (bias pair, fused shortcut segment, GroupNorm sums,
residual, fp32 outputs of 3 and 18 channels, partial boxes, strided data gradient). Results are compared with torch in
fp32 (TF32 off) on the same bf16 operands, and two calls must give the same bits."""
import zlib

import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda'
WS_BYTES = 24 << 20          # the step scope's split-K workspace (ops.StepScope.workspace)
BF16_HALF_ULP = 2.0 ** -8    # largest relative rounding error of a bf16 output


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(name):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(f'conv_pingpong_{name}'.encode()))


def _rand(g, shape, scale=1.0):
    return ((torch.rand(shape, generator=g, device=DEV) * 2 - 1) * scale).to(torch.bfloat16)


def _no_tf32(fn):
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _conv_ref(x, w, k, pads, stride=(1, 1, 1)):
    """fp32 convolution of channels-last x with packed w [cout][tap][cin] and (front t, h, w) padding; returns NCDHW."""
    cout, cin = w.shape[0], x.shape[-1]
    wt = w.float().reshape(cout, k, k, k, cin).permute(0, 4, 1, 2, 3)
    pt, ph, pw = pads
    return F.conv3d(F.pad(x.float().permute(0, 4, 1, 2, 3), (pw, pw, ph, ph, pt, 0)), wt, stride=stride)


def _fwd(x, w, k, cout, bias0=None, bias1=None, x1=None, residual=None, out_f32=False, sums=False, ws_bytes=WS_BYTES):
    """og_conv3d_fwd: (out, GroupNorm sums or None)."""
    from open_genie_b200 import _lib
    N, T, H, W, cin = x.shape
    c1 = x1.shape[-1] if x1 is not None else 0
    out = torch.empty((N, T, H, W, cout), dtype=torch.float32 if out_f32 else torch.bfloat16, device=DEV)
    gs = torch.zeros((N, 2), dtype=torch.float64, device=DEV) if sums else None
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    pad = (k - 1) // 2
    _lib.call('og_conv3d_fwd', x.data_ptr(), cin, k, k, k, k - 1, pad, pad, p(x1), c1, w.data_ptr(), w.shape[1], p(bias0),
              p(bias1), p(residual), out.data_ptr(), int(out_f32), N, T, H, W, cout, ws.data_ptr() if ws_bytes else None,
              ws_bytes, p(gs), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out, gs


def _dgrad(dy, w, k, cin, out_f32=False, ws_bytes=WS_BYTES):
    from open_genie_b200 import _lib
    N, T, H, W, cout = dy.shape
    dx = torch.empty((N, T, H, W, cin), dtype=torch.float32 if out_f32 else torch.bfloat16, device=DEV)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    pad = (k - 1) // 2
    _lib.call('og_conv3d_dgrad', dy.data_ptr(), cout, w.shape[0], w.data_ptr(), w.shape[1], 0, k, k, k, k - 1, pad, pad,
              dx.data_ptr(), int(out_f32), N, T, H, W, cin, ws.data_ptr() if ws_bytes else None, ws_bytes,
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dx


def _dgrad_ref(dy, w, k, in_shape, pads, stride=(1, 1, 1)):
    """Input gradient of _conv_ref by autograd, channels last."""
    x = torch.zeros(in_shape, device=DEV, requires_grad=True)

    def run():
        y = _conv_ref(x, w, k, pads, stride)
        y.backward(dy.float().permute(0, 4, 1, 2, 3))
        return x.grad
    return _no_tf32(run)


def _check_fwd(name, out, ref, sums, out2, sums2=None):
    assert_close(out, ref, 2e-3 + BF16_HALF_ULP, 1e-3 * ref.abs().max().item(), f'{name} forward')
    if sums is not None:
        N = out.shape[0]
        y = out.double().reshape(N, -1)
        assert torch.all((sums[:, 0] - y.sum(1)).abs() <= 1e-4 * y.abs().sum(1)), f'{name}: GroupNorm sum'
        assert torch.all((sums[:, 1] - (y * y).sum(1)).abs() <= 1e-4 * (y * y).sum(1)), f'{name}: GroupNorm sum of squares'
    assert torch.equal(out, out2), f'{name}: two calls differ'


@pytest.mark.parametrize('items', ['one_per_cta', 'grid_plus_one', 'three_per_cta_plus_one'])
def test_item_counts(items):
    """Forward (bias, GroupNorm sums) and data gradient with 128 x 1 x 1 voxel tiles, one tile per W row: the launch has
    exactly `rows` items of 27 k-blocks, a count that does not divide the stage ring."""
    sms = _sms()
    rows = {'one_per_cta': sms // 2, 'grid_plus_one': sms + 1, 'three_per_cta_plus_one': 3 * sms + 1}[items]
    C, k = 64, 3
    g = _gen(items)
    x = _rand(g, (1, 1, rows, 128, C))
    dy = _rand(g, (1, 1, rows, 128, C))
    w = _rand(g, (C, k ** 3 * C), 0.2)
    bias = torch.rand(C, generator=g, device=DEV) * 2 - 1
    out, sums = _fwd(x, w, k, C, bias0=bias, sums=True)
    out2, _ = _fwd(x, w, k, C, bias0=bias, sums=True)
    ref = _no_tf32(lambda: _conv_ref(x, w, k, (2, 1, 1)) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd(items, out, ref, sums, out2)
    dx = _dgrad(dy, w, k, C)
    ref_dx = _dgrad_ref(dy, w, k, x.shape[:4] + (C,), (2, 1, 1))
    assert_close(dx, ref_dx, 2e-3 + BF16_HALF_ULP, 1e-3 * ref_dx.abs().max().item(), f'{items} data gradient')
    assert torch.equal(dx, _dgrad(dy, w, k, C)), f'{items}: two data-gradient calls differ'


def test_idle_second_consumer_512():
    """512 -> 512 @ 4x8x8 at batch 2 without workspace: 16 tiles, so every CTA has one item."""
    C, k, N = 512, 3, 2
    g = _gen('idle512')
    x = _rand(g, (N, 4, 8, 8, C))
    dy = _rand(g, (N, 4, 8, 8, C))
    w = _rand(g, (C, k ** 3 * C), 0.05)
    bias = torch.rand(C, generator=g, device=DEV) * 2 - 1
    out, sums = _fwd(x, w, k, C, bias0=bias, sums=True, ws_bytes=0)
    out2, _ = _fwd(x, w, k, C, bias0=bias, sums=True, ws_bytes=0)
    ref = _no_tf32(lambda: _conv_ref(x, w, k, (2, 1, 1)) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd('idle 512', out, ref, sums, out2)
    dx = _dgrad(dy, w, k, C, out_f32=True, ws_bytes=0)
    ref_dx = _dgrad_ref(dy, w, k, x.shape, (2, 1, 1))
    assert_close(dx, ref_dx, 2e-3, 1e-3 * ref_dx.abs().max().item(), 'idle 512 data gradient')
    assert torch.equal(dx, _dgrad(dy, w, k, C, out_f32=True, ws_bytes=0)), 'idle 512: two data-gradient calls differ'


def test_split_items_of_unequal_length():
    """192 -> 128 channels, 3x3x3: 81 k-blocks split 8 ways (16 tiles), so the split items have 10 or 11 k-blocks."""
    Ci, Co, k, N = 192, 128, 3, 2
    g = _gen('split_unequal')
    x = _rand(g, (N, 16, 8, 8, Ci))
    dy = _rand(g, (N, 16, 8, 8, Co))
    w = _rand(g, (Co, k ** 3 * Ci), 0.1)
    bias = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    from open_genie_b200 import _lib
    n0 = _lib.launch_count()
    out, sums = _fwd(x, w, k, Co, bias0=bias, sums=True)
    assert _lib.launch_count() - n0 == 2, 'the forward was not split'
    out2, _ = _fwd(x, w, k, Co, bias0=bias, sums=True)
    ref = _no_tf32(lambda: _conv_ref(x, w, k, (2, 1, 1)) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd('split', out, ref, sums, out2)
    # data gradient: 128 output channels = 2 k-blocks per tap, 54 k-blocks; dx fp32
    wd = _rand(g, (Ci, k ** 3 * Co), 0.1)    # a 128 -> 192 convolution's weights: its data gradient has 192 outputs
    dyd = _rand(g, (N, 16, 8, 8, Ci))
    dx = _dgrad(dyd, wd, k, Co, out_f32=True)
    ref_dx = _dgrad_ref(dyd, wd, k, (N, 16, 8, 8, Co), (2, 1, 1))
    assert_close(dx, ref_dx, 2e-3, 1e-3 * ref_dx.abs().max().item(), 'split data gradient')
    assert torch.equal(dx, _dgrad(dyd, wd, k, Co, out_f32=True)), 'split: two data-gradient calls differ'


def test_fused_shortcut_bias_pair_groupnorm():
    """3x3x3 over 128 channels + the 1x1x1 shortcut over 64 channels in one accumulator, bias0 + bias1, GroupNorm sums."""
    C0, C1, Co, k, N = 128, 64, 128, 3, 2
    g = _gen('fused')
    x0 = _rand(g, (N, 4, 16, 16, C0))
    x1 = _rand(g, (N, 4, 16, 16, C1))
    w = _rand(g, (Co, k ** 3 * C0 + C1), 0.1)
    b0 = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    b1 = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    out, sums = _fwd(x0, w, k, Co, bias0=b0, bias1=b1, x1=x1, sums=True)
    out2, _ = _fwd(x0, w, k, Co, bias0=b0, bias1=b1, x1=x1, sums=True)

    def ref():
        y = _conv_ref(x0, w[:, :k ** 3 * C0], k, (2, 1, 1))
        y = y + torch.einsum('nthwc,oc->nothw', x1.float(), w[:, k ** 3 * C0:].float())
        return (y + (b0 + b1).view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd('fused shortcut', out, _no_tf32(ref), sums, out2)


@pytest.mark.parametrize('out_kind', ['bf16_staged', 'fp32', 'bf16_96_channels'])
def test_residual(out_kind):
    """out = conv + bias + residual: through the staged bf16 stores, and through the masked fragment stores."""
    Ci, k, N = 64, 3, 2
    Co = 96 if out_kind == 'bf16_96_channels' else 128
    g = _gen(f'residual_{out_kind}')
    x = _rand(g, (N, 4, 12, 20, Ci))      # partial boxes along h and w
    w = _rand(g, (Co, k ** 3 * Ci), 0.1)
    res = _rand(g, (N, 4, 12, 20, Co))
    bias = torch.rand(Co, generator=g, device=DEV) * 2 - 1
    f32 = out_kind == 'fp32'
    out, _ = _fwd(x, w, k, Co, bias0=bias, residual=res, out_f32=f32)
    out2, _ = _fwd(x, w, k, Co, bias0=bias, residual=res, out_f32=f32)
    ref = _no_tf32(lambda: _conv_ref(x, w, k, (2, 1, 1)) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1) + res.float()
    _check_fwd(f'residual {out_kind}', out, ref, None, out2)


@pytest.mark.parametrize('cout,k', [(3, 3), (18, 1)])
def test_narrow_fp32_outputs(cout, k):
    """The tokenizer's fp32 tail (128 -> 3, BN = 16) and head (512 -> 18, 1x1x1, BN = 32)."""
    Ci = 128 if cout == 3 else 512
    N = 2
    g = _gen(f'narrow_{cout}')
    x = _rand(g, (N, 4, 8, 8, Ci))
    w = _rand(g, (cout, k ** 3 * Ci), 0.1)
    bias = torch.rand(cout, generator=g, device=DEV) * 2 - 1
    out, _ = _fwd(x, w, k, cout, bias0=bias, out_f32=True)
    out2, _ = _fwd(x, w, k, cout, bias0=bias, out_f32=True)
    pads = (k - 1, (k - 1) // 2, (k - 1) // 2)
    ref = _no_tf32(lambda: _conv_ref(x, w, k, pads) + bias.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    _check_fwd(f'fp32 {cout} channels', out, ref, None, out2)


@pytest.mark.parametrize('out_f32', [False, True])
def test_mn_major_dgrad_partial_boxes(out_f32):
    """Data gradient (MN-major weights) on a 3 x 10 x 12 grid: the 16 x 8 x 1 voxel boxes overhang along w and h."""
    Ci, Co, k, N = 128, 64, 3, 2
    g = _gen(f'dgrad_partial_{out_f32}')
    dy = _rand(g, (N, 3, 10, 12, Co))
    w = _rand(g, (Co, k ** 3 * Ci), 0.1)
    dx = _dgrad(dy, w, k, Ci, out_f32=out_f32)
    ref = _dgrad_ref(dy, w, k, (N, 3, 10, 12, Ci), (2, 1, 1))
    tol = 2e-3 if out_f32 else 2e-3 + BF16_HALF_ULP
    assert_close(dx, ref, tol, 1e-3 * ref.abs().max().item(), 'partial-box data gradient')
    assert torch.equal(dx, _dgrad(dy, w, k, Ci, out_f32=out_f32)), 'partial-box data gradient: two calls differ'


@pytest.mark.parametrize('stride', [(1, 2, 2), (2, 2, 2)])
def test_strided_dgrad(stride):
    """og_conv3d_strided_dgrad: one launch per residue class of the input grid, rows stored at stride s into dx."""
    from open_genie_b200 import _lib
    Ci, Co, k, N, T, H, W = 128, 128, 3, 2, 8, 16, 16
    st, sh, sw = stride
    pt, ph = k - 1 + (1 - st), 1
    To, Ho, Wo = (T + pt - k) // st + 1, (H + 2 * ph - k) // sh + 1, (W + 2 * ph - k) // sw + 1
    g = _gen(f'strided_{stride}')
    dy = _rand(g, (N, To, Ho, Wo, Co))
    w = _rand(g, (Co, k ** 3 * Ci), 0.1)

    def call():
        dx = torch.empty((N, T, H, W, Ci), dtype=torch.bfloat16, device=DEV)
        _lib.call('og_conv3d_strided_dgrad', dy.data_ptr(), Co, Co, w.data_ptr(), w.shape[1], k, k, k, st, sh, sw, pt, ph,
                  ph, dx.data_ptr(), N, T, H, W, Ci, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return dx
    dx = call()
    ref = _dgrad_ref(dy, w, k, (N, T, H, W, Ci), (pt, ph, ph), stride)
    assert_close(dx, ref, 2e-3 + BF16_HALF_ULP, 1e-3 * ref.abs().max().item(), f'strided {stride} data gradient')
    assert torch.equal(dx, call()), f'strided {stride}: two calls differ'
