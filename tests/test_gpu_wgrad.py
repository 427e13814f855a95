"""The weight-gradient kernel through the C ABI at the benchmark's shapes (batch 8): dW (and db) against an fp32 GPU
reference on the same bf16 operands, run-to-run bit identity of the stream-K reduction, and the reduced-workspace
fallbacks (no workspace, one slot)."""
import zlib

import pytest
import torch

from helpers import assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda'
SCRATCH_BYTES = 64 << 20     # the step scope's reduction scratch (ops.StepScope.scratch)
SLOT_BYTES = 128 * 256 * 4   # one 128 x 256 fp32 partial tile


def _operands(seed, N, cin, cout, T, H, W, To, Ho, Wo):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.rand((N, T, H, W, cin), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    dy = (torch.rand((N, To, Ho, Wo, cout), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    return x, dy


def _wgrad(x, dy, cout, k, stride, ws_bytes, n_bias=0):
    """dW as [cout][tap][cin] fp32 (and db[:n_bias]) from og_conv3d_wgrad / _bias / _strided_wgrad."""
    from open_genie_b200 import _lib
    N, T, H, W, cin = x.shape
    _, To, Ho, Wo, _ = dy.shape
    dw = torch.zeros((cout, k ** 3 * cin), dtype=torch.float32, device=DEV)
    db = torch.zeros(max(n_bias, 1), dtype=torch.float32, device=DEV)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    wsp = ws.data_ptr() if ws_bytes else None
    s = torch.cuda.current_stream().cuda_stream
    p = k // 2
    if stride != 1:
        _lib.call('og_conv3d_strided_wgrad', dy.data_ptr(), cout, x.data_ptr(), cin, dw.data_ptr(), dw.shape[1], k, k, k,
                  stride, stride, stride, p, p, p, N, T, H, W, wsp, ws_bytes, s)
    elif n_bias:
        _lib.call('og_conv3d_wgrad_bias', dy.data_ptr(), cout, x.data_ptr(), cin, dw.data_ptr(), dw.shape[1], k, k, k,
                  p, p, p, N, T, H, W, db.data_ptr(), n_bias, wsp, ws_bytes, s)
    else:
        _lib.call('og_conv3d_wgrad', dy.data_ptr(), cout, x.data_ptr(), cin, dw.data_ptr(), dw.shape[1], k, k, k,
                  p, p, p, N, T, H, W, wsp, ws_bytes, s)
    torch.cuda.synchronize()
    return dw, db[:n_bias]


def _reference(x, dy, cout, k, stride):
    """torch's fp32 weight gradient (TF32 off) of the same bf16 operands, in the kernel's [cout][tap][cin] order."""
    xf = x.float().permute(0, 4, 1, 2, 3)
    dyf = dy.float().permute(0, 4, 1, 2, 3)
    cin = x.shape[-1]
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        w = torch.nn.grad.conv3d_weight(xf, (cout, cin, k, k, k), dyf, stride=stride, padding=k // 2)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return w.permute(0, 2, 3, 4, 1).reshape(cout, -1), dyf.sum(dim=(0, 2, 3, 4))


# (N, cin, cout, T, H, W, kernel, stride, n_bias)
SHAPES = {
    '128to128_16x64x64': (8, 128, 128, 16, 64, 64, 3, 1, 0),
    '256to256_16x32x32': (8, 256, 256, 16, 32, 32, 3, 1, 0),
    '512to512_4x8x8': (8, 512, 512, 4, 8, 8, 3, 1, 0),
    '512to4096_4x8x8': (8, 512, 4096, 4, 8, 8, 3, 1, 0),
    '256to1024_16x32x32': (8, 256, 1024, 16, 32, 32, 3, 1, 0),
    'strided_256_16x32x32': (8, 256, 256, 16, 32, 32, 3, 2, 0),
    'bias_256to256_8x16x16': (8, 256, 256, 8, 16, 16, 3, 1, 250),
    'ragged_cin64_bias': (3, 64, 72, 5, 7, 9, 3, 1, 70),
}


def _case(name):
    N, cin, cout, T, H, W, k, stride, n_bias = SHAPES[name]
    To, Ho, Wo = ((d + 2 * (k // 2) - k) // stride + 1 for d in (T, H, W))
    x, dy = _operands(zlib.crc32(name.encode()), N, cin, cout, T, H, W, To, Ho, Wo)
    return x, dy, cout, k, stride, n_bias


@pytest.mark.parametrize('name', list(SHAPES))
def test_wgrad_matches_fp32_reference(name):
    x, dy, cout, k, stride, n_bias = _case(name)
    dw, db = _wgrad(x, dy, cout, k, stride, SCRATCH_BYTES, n_bias)
    ref_w, ref_b = _reference(x, dy, cout, k, stride)
    assert_close(dw, ref_w, 2e-3, 1e-3 * ref_w.abs().max().item(), f'{name} dW')
    if n_bias:
        assert_close(db, ref_b[:n_bias], 2e-3, 1e-3 * ref_b.abs().max().item(), f'{name} db')
    # stream-K: the cut tiles are summed in a fixed order, so a second call gives the same bits
    dw2, db2 = _wgrad(x, dy, cout, k, stride, SCRATCH_BYTES, n_bias)
    assert torch.equal(dw, dw2) and torch.equal(db, db2), f'{name}: two calls differ'


@pytest.mark.parametrize('name', ['256to256_16x32x32', 'ragged_cin64_bias'])
@pytest.mark.parametrize('ws_bytes', [0, SLOT_BYTES + 128 * 4])
def test_wgrad_small_workspace(name, ws_bytes):
    """Without room for a slot per share the work falls back to whole tiles per CTA: same answer, no workspace."""
    x, dy, cout, k, stride, n_bias = _case(name)
    dw, db = _wgrad(x, dy, cout, k, stride, ws_bytes, n_bias)
    ref_w, ref_b = _reference(x, dy, cout, k, stride)
    assert_close(dw, ref_w, 2e-3, 1e-3 * ref_w.abs().max().item(), f'{name} dW, {ws_bytes} B workspace')
    if n_bias:
        assert_close(db, ref_b[:n_bias], 2e-3, 1e-3 * ref_b.abs().max().item(), f'{name} db, {ws_bytes} B workspace')
