"""The convolution forward and data gradient through the C ABI at the benchmark's deepest stage (512 -> 512, 3x3x3 @ 4x8x8),
whose tiles cannot fill the SMs, so the K loop is split over one workspace slab per split: results against an fp32 GPU
reference on the same bf16 operands, run-to-run bit identity, and the split shrinking to the slabs the workspace holds
(batch 8: 64 tiles, split 2; batch 2: 16 tiles, split 8)."""
import zlib

import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda'
C, K, T, H, W = 512, 3, 4, 8, 8
FULL_BYTES = 24 << 20        # the step scope's split-K workspace (ops.StepScope.workspace)
BF16_HALF_ULP = 2.0 ** -8    # largest relative rounding error of a bf16 output


def _slab_bytes(N):
    return N * T * H * W * C * 4


def _operands(N):
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'conv_splitk_{N}'.encode()))
    x = (torch.rand((N, T, H, W, C), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    dy = (torch.rand((N, T, H, W, C), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    w = (torch.rand((C, C, K, K, K), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)    # (cout, cin, kt, kh, kw)
    bias = torch.rand(C, generator=g, device=DEV) * 2 - 1
    packed = w.permute(0, 2, 3, 4, 1).reshape(C, -1).contiguous()                           # [cout][tap][cin]
    return x, dy, w, packed, bias


def _workspace(ws_bytes):
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    return ws, (ws.data_ptr() if ws_bytes else None)


def _fwd(x, packed, bias, ws_bytes):
    """og_conv3d_fwd with bias and GroupNorm sums: (bf16 out, fp64 sums [N][2], kernels launched)."""
    from open_genie_b200 import _lib
    N = x.shape[0]
    out = torch.empty((N, T, H, W, C), dtype=torch.bfloat16, device=DEV)
    sums = torch.zeros((N, 2), dtype=torch.float64, device=DEV)
    ws, wsp = _workspace(ws_bytes)
    n0 = _lib.launch_count()
    _lib.call('og_conv3d_fwd', x.data_ptr(), C, K, K, K, 1, 1, 1, None, 0, packed.data_ptr(), packed.shape[1],
              bias.data_ptr(), None, None, out.data_ptr(), 0, N, T, H, W, C, wsp, ws_bytes, sums.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out, sums, _lib.launch_count() - n0


def _dgrad(dy, packed, ws_bytes):
    """og_conv3d_dgrad with an fp32 dx: (dx, kernels launched)."""
    from open_genie_b200 import _lib
    N = dy.shape[0]
    dx = torch.empty((N, T, H, W, C), dtype=torch.float32, device=DEV)
    ws, wsp = _workspace(ws_bytes)
    n0 = _lib.launch_count()
    _lib.call('og_conv3d_dgrad', dy.data_ptr(), C, C, packed.data_ptr(), packed.shape[1], 0, K, K, K, 1, 1, 1,
              dx.data_ptr(), 1, N, T, H, W, C, wsp, ws_bytes, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dx, _lib.launch_count() - n0


def _reference(x, dy, w, bias):
    """torch's fp32 forward and input gradient (TF32 off) of the same bf16 operands, channels last."""
    N = x.shape[0]
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        out = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w.float(), bias, padding=1)
        dx = torch.nn.grad.conv3d_input((N, C, T, H, W), w.float(), dy.float().permute(0, 4, 1, 2, 3), padding=1)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out.permute(0, 2, 3, 4, 1), dx.permute(0, 2, 3, 4, 1)


@pytest.mark.parametrize('N', [8, 2])
@pytest.mark.parametrize('workspace', ['full', 'two_slabs', 'one_slab', 'none'])
def test_conv_split_k_matches_fp32_reference(N, workspace):
    ws_bytes = {'full': FULL_BYTES, 'two_slabs': 2 * _slab_bytes(N), 'one_slab': _slab_bytes(N), 'none': 0}[workspace]
    launches = 2 if workspace in ('full', 'two_slabs') else 1     # split: the GEMM and the finish pass; unsplit: the GEMM
    x, dy, w, packed, bias = _operands(N)
    ref_out, ref_dx = _reference(x, dy, w, bias)
    name = f'N={N}, {workspace} workspace'

    out, sums, n = _fwd(x, packed, bias, ws_bytes)
    assert n == launches, f'{name}: forward launched {n} kernels'
    # the tolerances of the weight-gradient test, plus the output's own bf16 rounding
    assert_close(out, ref_out, 2e-3 + BF16_HALF_ULP, 1e-3 * ref_out.abs().max().item(), f'{name} forward')
    y = out.double().reshape(N, -1)
    assert torch.all((sums[:, 0] - y.sum(1)).abs() <= 1e-4 * y.abs().sum(1)), f'{name}: GroupNorm sum'
    assert torch.all((sums[:, 1] - (y * y).sum(1)).abs() <= 1e-4 * (y * y).sum(1)), f'{name}: GroupNorm sum of squares'

    dx, n = _dgrad(dy, packed, ws_bytes)
    assert n == launches, f'{name}: data gradient launched {n} kernels'
    assert_close(dx, ref_dx, 2e-3, 1e-3 * ref_dx.abs().max().item(), f'{name} data gradient')

    # the slabs are added in split order, so a second call gives the same bits
    out2, _, _ = _fwd(x, packed, bias, ws_bytes)
    dx2, _ = _dgrad(dy, packed, ws_bytes)
    assert torch.equal(out, out2) and torch.equal(dx, dx2), f'{name}: two calls differ'
