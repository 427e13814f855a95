"""Every path of the layout kernels (csrc/layout.cu) and of the fused AdamW (csrc/optim.cu) against exact and float64
references, element by element.

Paths covered:
- og_pixel_shuffle3d in both directions on each of its five kernels: og_pixel_shuffle_vec_kernel<8>, <4> and <2>
  (c % 8 == 0, p*q*r in {2, 4, 8}, x and y 16-byte aligned), the generic og_pixel_shuffle_kernel (any other p*q*r, or
  x off alignment) and og_pixel_shuffle_scalar_kernel (c % 8 != 0, or y off alignment), with grid-stride sizes.
- Bit exact (pure data movement, or one IEEE operation done the same way in torch): the NCDHW <-> NDHWC casts in fp32
  and bf16, og_pad_channels, og_copy_rows_to_bf16, og_sub_rows, og_frames_u8_to_video and og_maxpool2x2 (NaN
  included). Where a NaN is expected only its position is compared: CUDA and torch use different payloads.
- float64 references with per-element worst-case bounds: og_colsum (vector and scalar kernel), og_mse_fwd /
  og_mse_bwd, og_sqdiff_sum, og_blurpool3d / og_blurpool2d forward and backward.
- og_adamw_step through a hand-built, shuffled chunk table: vector chunks and scalar tails, a parameter off alignment,
  gradient or bf16 destination absent, pitched and offset bf16 destinations, host and device step count, device
  learning rate and gradient scale; float64 state with an error bound carried across the steps. FusedAdamW on each
  form of bf16 operand target.

Every output sits in a `Guarded` buffer, so an element the kernel does not write, or a write past the end, fails.
Accumulated outputs start from non-zero values. The `test_bound(s)_reject_*` tests run on the CPU and show that each
bound still rejects the mistakes it exists to catch; the branch mirrors and the argument validation run on the CPU too.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import Guarded

GPU = pytest.mark.gpu
DEV = 'cuda'
BF16, F32T, F64T = torch.bfloat16, torch.float32, torch.float64

# Rounding model, as in test_gpu_attention_paths.py. U is the unit roundoff of bf16 (8 significant bits). F32 is one
# fp32 ulp, used per operation (twice fp32's unit roundoff); a sum of n terms in any order whose every term passes
# through at most d roundings is within gam(d) of the exact sum, relative to the sum of the terms' magnitudes.
U = 2.0 ** -8
F32 = 2.0 ** -23
SLACK = 1.02    # second-order terms (an error that is itself rounded, U * err) are folded into this factor
# powf: maximum error 4 ulp (CUDA C++ Programming Guide, single-precision mathematical functions). The device-side
# bias corrections 1 - powf(beta, t) carry it, amplified by beta^t / (1 - beta^t).
POWF_ULP = 4
CAPPED_THREADS = 132 * 32 * 256     # ew_blocks caps an elementwise grid at 32 blocks of 256 threads per SM (132 SMs)


def gam(n):
    return n * F32


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def cdiv(a, b):
    return -(-a // b)


def f32(x):
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------------------------
ITY = {BF16: torch.int16, F32T: torch.int32}


def check_bits(name, got, ref, nan_any=False):
    """Bit equality. With nan_any a NaN only has to meet a NaN (payloads differ between CUDA and torch)."""
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape, got.dtype, ref.dtype)
    got, ref = got.contiguous(), ref.contiguous()
    bad = got.view(ITY[got.dtype]) != ref.view(ITY[ref.dtype])
    if nan_any:
        gn, rn = torch.isnan(got), torch.isnan(ref)
        bad = (bad & ~(gn & rn)) | (gn != rn)
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f'{name}: {int(bad.sum())}/{bad.numel()} elements differ; first at flat {i}: got '
                             f'{got.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r}')


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


def _rejects(fn):
    with pytest.raises(AssertionError):
        fn()


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _gen(seed, device=DEV):
    return torch.Generator(device=device).manual_seed(seed)


def _rand(shape, seed, amp=1.0, dtype=BF16, device=DEV):
    return (torch.randn(shape, generator=_gen(seed, device), device=device) * amp).to(dtype)


def _bits(shape, seed):
    """bf16 tensor of random bit patterns (NaNs and infinities included): data movement must keep every bit."""
    r = torch.randint(-2 ** 15, 2 ** 15, shape, generator=_gen(seed), device=DEV, dtype=torch.int32)
    return r.to(torch.int16).view(BF16)


def _placed(t, offset):
    """A copy of t placed `offset` elements into a fresh (256-byte aligned) buffer."""
    b = torch.empty(t.numel() + offset, dtype=t.dtype, device=t.device)
    v = b[offset:].view(t.shape)
    v.copy_(t)
    return v


def _kernels_run(fn):
    """Names of the kernels two calls of `fn` launch (see test_gpu_attention_paths._kernels_run)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


# ------------------------------------------------------------------------------------------------------------------
# pixel shuffle
# ------------------------------------------------------------------------------------------------------------------
PS_CASES = {
    # name: (N, T, H, W, c, p, q, r, x offset, y offset in elements)
    'vec8_c8': (3, 3, 5, 7, 8, 2, 2, 2, 0, 0),
    'vec8_c64': (1, 1, 3, 5, 64, 2, 2, 2, 0, 0),
    'vec8_c256': (2, 3, 3, 1, 256, 2, 2, 2, 0, 0),
    'vec8_grid_stride': (1, 3, 211, 215, 64, 2, 2, 2, 0, 0),
    'vec4_c64': (3, 1, 5, 3, 64, 1, 2, 2, 0, 0),
    'vec4_c128': (1, 3, 7, 5, 128, 1, 2, 2, 0, 0),
    'vec2_c8': (3, 5, 3, 7, 8, 2, 1, 1, 0, 0),
    'generic_144_c8': (3, 3, 5, 3, 8, 1, 4, 4, 0, 0),
    'generic_111_c64': (3, 1, 5, 7, 64, 1, 1, 1, 0, 0),
    'generic_333_c8': (1, 3, 3, 5, 8, 3, 3, 3, 0, 0),
    'generic_x_off': (3, 3, 5, 1, 64, 2, 2, 2, 1, 0),
    'scalar_144_c3': (3, 1, 5, 7, 3, 1, 4, 4, 0, 0),
    'scalar_222_c1': (1, 3, 5, 3, 1, 2, 2, 2, 0, 0),
    'scalar_122_c12': (3, 3, 1, 5, 12, 1, 2, 2, 0, 0),
    'scalar_y_off': (3, 3, 5, 1, 64, 2, 2, 2, 0, 1),
    'scalar_grid_stride': (1, 5, 80, 80, 3, 1, 4, 4, 0, 0),
}
PS_KERNELS = ('og_pixel_shuffle_vec_kernel<8>', 'og_pixel_shuffle_vec_kernel<4>', 'og_pixel_shuffle_vec_kernel<2>',
              'og_pixel_shuffle_kernel(', 'og_pixel_shuffle_scalar_kernel')


def ps_plan(N, T, H, W, c, p, q, r, xo, yo):
    """(kernel, work items) og_pixel_shuffle3d dispatches to (offsets in bf16 elements from 16-byte aligned bases)."""
    pqr = p * q * r
    if c % 8 or yo % 8:
        return 'og_pixel_shuffle_scalar_kernel', N * T * H * W * pqr * c
    if xo % 8 == 0 and pqr in (2, 4, 8):
        return f'og_pixel_shuffle_vec_kernel<{pqr}>', N * T * H * W * (c // 8)
    return 'og_pixel_shuffle_kernel(', N * T * H * W * pqr * (c // 8)


def ps_ref(x, N, T, H, W, c, p, q, r):
    return x.view(N, T, H, W, c, p, q, r).permute(0, 1, 5, 2, 6, 3, 7, 4).reshape(N, T * p, H * q, W * r, c)


def test_pixel_shuffle_plan_covers_every_kernel():
    plans = {k: ps_plan(*v) for k, v in PS_CASES.items()}
    assert {k for k, _ in plans.values()} == set(PS_KERNELS)
    by_prefix = {'vec8': PS_KERNELS[0], 'vec4': PS_KERNELS[1], 'vec2': PS_KERNELS[2], 'generic': PS_KERNELS[3],
                 'scalar': PS_KERNELS[4]}
    for name, (kern, items) in plans.items():
        assert kern == by_prefix[name.split('_')[0]], (name, kern)
        if name.endswith('grid_stride'):
            assert items > CAPPED_THREADS, (name, items)


def pixel_shuffle_run(case, seed):
    N, T, H, W, c, p, q, r, xo, yo = PS_CASES[case]
    xshape, yshape = (N, T, H, W, c * p * q * r), (N, T * p, H * q, W * r, c)
    x = _placed(_bits(xshape, seed), xo)
    y = Guarded(yshape, BF16, offset=yo)
    _call('og_pixel_shuffle3d', x.data_ptr(), y.ptr(), 0, N, T, H, W, c, p, q, r)
    back = Guarded(xshape, BF16, offset=xo)
    _call('og_pixel_shuffle3d', back.ptr(), y.ptr(), 1, N, T, H, W, c, p, q, r)
    return x, y, back


@GPU
@pytest.mark.parametrize('case', sorted(PS_CASES))
def test_pixel_shuffle(case):
    """Forward against the view/permute reference, and inverse(forward(x)) == x, bit for bit, guards intact."""
    N, T, H, W, c, p, q, r, _, _ = PS_CASES[case]
    x, y, back = pixel_shuffle_run(case, 100 + len(case))
    torch.cuda.synchronize()
    y.check_guard('y')
    back.check_guard('inverse')
    check_bits('y', y.t, ps_ref(x, N, T, H, W, c, p, q, r))
    check_bits('inverse(forward(x))', back.t, x)


# ------------------------------------------------------------------------------------------------------------------
# NCDHW <-> NDHWC casts, channel padding, row copies, subtraction, frames, max-pool: bit exact
# ------------------------------------------------------------------------------------------------------------------
SPECIALS = [0.0, -0.0, math.inf, -math.inf, math.nan, 1e-40, -3e-39, 1.4e-45, 1 + 2 ** -8, 1 + 3 * 2 ** -8,
            -(1 + 2 ** -8), -(1 + 3 * 2 ** -8), 1 + 2 ** -8 + 2 ** -22, 3.3895314e38, 1e-45 * 3]


def _cast_values(shape, seed):
    """fp32 values: normal draws, with the specials (signed zeros, infinities, NaN, subnormals, bf16 rounding ties and
    their neighbours, a value that rounds to bf16 infinity) placed at spread positions."""
    x = _rand(shape, seed, 3.0, F32T).flatten()
    s = torch.tensor(SPECIALS, dtype=F32T, device=DEV)
    idx = torch.randperm(x.numel(), generator=_gen(seed + 1), device=DEV)[:min(x.numel(), 4 * len(SPECIALS))]
    x[idx] = s.repeat(4)[:idx.numel()]
    return x.view(shape)


CAST_SHAPES = [(N, C, V) for N in (1, 3) for C in (1, 3, 18, 32, 33, 96) for V in (1, 31, 32, 33, 1000)]


@GPU
@pytest.mark.parametrize('out_f32', [0, 1])
def test_ncdhw_to_ndhwc(out_f32):
    dt = F32T if out_f32 else BF16
    for i, (N, C, V) in enumerate(CAST_SHAPES):
        x = _cast_values((N, C, V), 200 + i)
        y = Guarded((N, V, C), dt)
        _call('og_ncdhw_f32_to_ndhwc', x.data_ptr(), y.ptr(), out_f32, N, C, V)
        torch.cuda.synchronize()
        y.check_guard(f'y {(N, C, V)}')
        check_bits(f'y {(N, C, V)}', y.t, x.permute(0, 2, 1).to(dt), nan_any=True)


@GPU
@pytest.mark.parametrize('x_f32', [0, 1])
def test_ndhwc_to_ncdhw(x_f32):
    for i, (N, C, V) in enumerate(CAST_SHAPES):
        x = _cast_values((N, V, C), 300 + i)
        if not x_f32:
            x = x.to(BF16)
        y = Guarded((N, C, V), F32T)
        _call('og_ndhwc_to_ncdhw_f32', x.data_ptr(), x_f32, y.ptr(), N, C, V)
        torch.cuda.synchronize()
        y.check_guard(f'y {(N, C, V)}')
        check_bits(f'y {(N, C, V)}', y.t, x.float().permute(0, 2, 1), nan_any=True)


@GPU
@pytest.mark.parametrize('x_f32', [0, 1])
def test_pad_channels(x_f32):
    """cd > cs zero pads (pad columns are +0 bits), cd == cs copies, cd < cs truncates."""
    rows = 1001
    for i, (cs, cd) in enumerate(((3, 64), (18, 24), (40, 40), (64, 18), (9, 3))):
        x = _cast_values((rows, cs), 400 + i)
        if not x_f32:
            x = x.to(BF16)
        y = Guarded((rows, cd), BF16)
        _call('og_pad_channels', x.data_ptr(), x_f32, y.ptr(), rows, cs, cd)
        ref = torch.zeros(rows, cd, dtype=BF16, device=DEV)
        k = min(cs, cd)
        ref[:, :k] = x[:, :k].to(BF16)
        torch.cuda.synchronize()
        y.check_guard('y')
        check_bits(f'pad {cs}->{cd}', y.t, ref, nan_any=True)


@GPU
@pytest.mark.parametrize('src_f32', [0, 1])
def test_copy_rows_to_bf16(src_f32):
    """Strided source and destination; the destination columns beyond `cols` keep their NaN bits."""
    for i, (rows, cols, src_ld, dst_ld) in enumerate(((37, 27, 27, 64), (37, 18, 40, 64), (5, 100, 128, 100),
                                                      (300, 3, 8, 64))):
        src = _cast_values((rows, src_ld), 500 + i)
        if not src_f32:
            src = src.to(BF16)
        dst = Guarded((rows, dst_ld), BF16)
        _call('og_copy_rows_to_bf16', src.data_ptr(), src_f32, src_ld, dst.ptr(), dst_ld, rows, cols)
        torch.cuda.synchronize()
        dst.check_guard('dst')
        check_bits('copied columns', dst.t[:, :cols], src[:, :cols].to(BF16), nan_any=True)
        nan_bits = Guarded.BITS[BF16][1]
        assert bool((dst.t[:, cols:].contiguous().view(torch.int16) == nan_bits).all()), 'pad columns were written'


@GPU
@pytest.mark.parametrize('n', [8, 8 * 1_100_000])
def test_sub_rows(n):
    """bf16(float(a) - float(b)): magnitudes 2^-20..2^20 apart, so the fp32 difference is not always exact."""
    assert n == 8 or n // 8 > CAPPED_THREADS
    g = _gen(600 + n % 1000)
    a = (torch.randn(n, generator=g, device=DEV) * 2.0 ** torch.randint(-20, 21, (n,), generator=g, device=DEV)).to(BF16)
    b = (torch.randn(n, generator=g, device=DEV) * 2.0 ** torch.randint(-20, 21, (n,), generator=g, device=DEV)).to(BF16)
    out = Guarded((n,), BF16)
    _call('og_sub_rows', a.data_ptr(), b.data_ptr(), out.ptr(), n)
    torch.cuda.synchronize()
    out.check_guard('out')
    check_bits('a - b', out.t, (a.float() - b.float()).to(BF16))


@GPU
def test_frames_u8_to_video_all_bytes():
    """All 256 byte values, RGB and BGR input, NCDHW fp32 and padded NDHWC bf16 output (pad columns exactly +0)."""
    N, T, H, W = 2, 3, 5, 9
    V = T * H * W
    vals = torch.arange(N * V * 3) % 256
    frames_cpu = vals[torch.randperm(vals.numel(), generator=torch.Generator().manual_seed(700))].to(torch.uint8)
    assert frames_cpu.unique().numel() == 256
    frames = frames_cpu.view(N, T, H, W, 3).to(DEV)
    for bgr in (0, 1):
        rgb = frames_cpu.view(N, V, 3).float() / 255.          # IEEE division on the CPU
        if bgr:
            rgb = rgb.flip(-1)
        for out_kind, cpad in ((0, 3), (1, 3), (1, 64)):
            if out_kind == 0:
                out = Guarded((N, 3, V), F32T)
                ref = rgb.permute(0, 2, 1).contiguous()
            else:
                out = Guarded((N, V, cpad), BF16)
                ref = torch.zeros(N, V, cpad, dtype=BF16)
                ref[..., :3] = rgb.to(BF16)
            _call('og_frames_u8_to_video', frames.data_ptr(), bgr, out.ptr(), out_kind, cpad, N, T, H, W)
            torch.cuda.synchronize()
            out.check_guard('out')
            check_bits(f'bgr={bgr} kind={out_kind} cpad={cpad}', out.t.cpu(), ref)


def maxpool_run(x):
    N, H, W, C = x.shape
    y = Guarded((N, H // 2, W // 2, C), BF16)
    _call('og_maxpool2x2', x.data_ptr(), y.ptr(), N, H, W, C)
    torch.cuda.synchronize()
    y.check_guard('y')
    return y.t


def maxpool_ref(x):
    return F.max_pool2d(x.permute(0, 3, 1, 2).float().cpu(), 2).permute(0, 2, 3, 1)


@GPU
@pytest.mark.parametrize('shape', [(2, 224, 224, 64), (1, 7, 9, 8), (3, 2, 2, 512)])
def test_maxpool2x2(shape):
    """Values equal to F.max_pool2d (+0 and -0 compare equal); (1, 7, 9) takes the floor of odd extents."""
    x = _rand(shape, 800 + shape[1])
    x.view(-1)[::97] = 0.0
    x.view(-1)[1::89] = -0.0
    got, ref = maxpool_run(x).float().cpu(), maxpool_ref(x)
    bad = got != ref
    assert not bad.any(), f'{int(bad.sum())}/{bad.numel()} differ'


@GPU
def test_maxpool2x2_propagates_nan():
    """A NaN in any of the four window slots gives NaN, as nn.MaxPool2d does."""
    N, H, W, C = 1, 4, 6, 16
    x = _rand((N, H, W, C), 810)
    nan = float('nan')
    x[0, 0, 0, 0] = nan         # top-left slot of window (0, 0)
    x[0, 0, 3, 1] = nan         # top-right of window (0, 1)
    x[0, 3, 4, 2] = nan         # bottom-left of window (1, 2)
    x[0, 1, 1, 9] = nan         # bottom-right of window (0, 0), channel 9 (second half of the vector)
    x[0, 2, 2, 3] = nan
    x[0, 3, 3, 3] = nan         # two NaNs in one window
    x[0, 2, 0, :] = float('inf')
    x[0, 2, 0, 5] = nan         # NaN next to +inf
    got, ref = maxpool_run(x).float().cpu(), maxpool_ref(x)
    assert int(torch.isnan(ref).sum()) == 6
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), torch.nonzero(torch.isnan(got) != torch.isnan(ref))
    keep = ~torch.isnan(ref)
    assert torch.equal(got[keep], ref[keep])


# ------------------------------------------------------------------------------------------------------------------
# column sums
# ------------------------------------------------------------------------------------------------------------------
COLSUM_CASES = {
    # name: (rows, C, ld, x offset in bf16 elements)
    'vec_1x8': (1, 8, 8, 0),
    'vec_63x64': (63, 64, 64, 0),
    'vec_524288x128': (524288, 128, 128, 0),
    'vec_C3_ld64': (1000, 3, 64, 0),
    'vec_two_col_blocks': (300, 4000, 4096, 0),
    'scalar_ld2104': (300, 2100, 2104, 0),
    'scalar_ld12': (777, 10, 12, 0),
    'scalar_x_off8B': (513, 64, 64, 4),
}


def colsum_plan(rows, C, ld, xo, sms):
    """(kernel, rounding depth of one term) of og_colsum: mirrors its launch arithmetic. Vector kernel: one thread sums
    ceil(rpb / lanes) rows, the block sums `lanes` partials, and nb blocks add into out (which holds init) with atomics.
    Scalar kernel: 256 rows per thread, then the atomics."""
    if ld % 8 == 0 and (ld <= 2048 or ld % 2048 == 0) and xo % 8 == 0:
        col_blocks = cdiv(ld, 2048)
        want = cdiv(4 * sms, col_blocks)
        groups = cdiv(rows, 64)
        want = max(min(want, groups), 1)
        rpb = cdiv(groups, want) * 64
        nb = cdiv(rows, rpb)
        lanes = 256 // (min(ld, 2048) // 8)
        return 'og_colsum_vec_kernel', cdiv(rpb, lanes) + lanes + nb
    return 'og_colsum_kernel(', 256 + cdiv(rows, 256)


def colsum_expect(x, C, init, depth):
    xs = x[:, :C].double()
    return init.double() + xs.sum(0), gam(depth) * (init.double().abs() + xs.abs().sum(0))


def test_colsum_plan_covers_both_kernels():
    for sms in (132, num_sms()):
        kern = {k: colsum_plan(*v, sms)[0] for k, v in COLSUM_CASES.items()}
        for k, v in kern.items():
            assert v == ('og_colsum_vec_kernel' if k.startswith('vec') else 'og_colsum_kernel('), (k, v)


def test_bound_rejects_colsum_mistakes():
    rows, C = 63, 64
    x = _rand((rows, C), 900, device='cpu')
    init = _rand((C,), 901, dtype=F32T, device='cpu')
    ref, tol = colsum_expect(x, C, init, colsum_plan(rows, C, C, 0, 132)[1])
    check('exact', (init.double() + x.double().sum(0)).float(), ref, tol)
    _rejects(lambda: check('init overwritten', x.double().sum(0).float(), ref, tol))
    _rejects(lambda: check('last row dropped', (init.double() + x[:-1].double().sum(0)).float(), ref, tol))
    _rejects(lambda: check('column shifted', (init.double() + x.double().roll(1, 1).sum(0)).float(), ref, tol))


def colsum_run(case, seed):
    rows, C, ld, xo = COLSUM_CASES[case]
    x = _placed(_rand((rows, ld), seed), xo)
    init = _rand((C,), seed + 1, 4.0, F32T)
    out = Guarded((C,), F32T, guard=256, init=init)
    _call('og_colsum', x.data_ptr(), rows, C, ld, out.ptr())
    return x, init, out


@GPU
@pytest.mark.parametrize('case', sorted(COLSUM_CASES))
def test_colsum(case):
    rows, C, ld, xo = COLSUM_CASES[case]
    x, init, out = colsum_run(case, 1000 + len(case))
    torch.cuda.synchronize()
    out.check_guard('out (columns >= C)')
    check('colsum', out.t, *colsum_expect(x, C, init, colsum_plan(rows, C, ld, xo, num_sms())[1]))


# ------------------------------------------------------------------------------------------------------------------
# mse and the feature-space squared difference
# ------------------------------------------------------------------------------------------------------------------
def ew_blocks(total, sms):
    return max(min(cdiv(total, 256), sms * 32), 1)


def mse_fwd_expect(rec, tgt, N, C, V, init, sms):
    """loss_sum = init + sum (rec - tgt)^2. A term: the fp32 difference and its square (2), its thread's fma chain, the
    warp and block shuffles (10) and the atomics of the blocks onto init."""
    d = rec.double().view(N, V, C).permute(0, 2, 1) - tgt.double().view(N, C, V)
    s = (d * d).sum()
    blocks = ew_blocks(N * C * V, sms)
    depth = 2 + cdiv(N * C * V, blocks * 256) + 10 + blocks
    return init + s, gam(depth) * (abs(init) + s)


def mse_bwd_expect(rec, tgt, gs, N, C, V, cpad, mut=()):
    """drec[n, v, c] = gs * 2 (rec - tgt) / (N C V) for c < C, exactly +0 in the pad columns. Rounding points: the fp32
    coefficient, gs * coefficient, rec - tgt, the product (4 fp32 roundings), the bf16 store."""
    r = rec.double().flatten()[:N * V * C].view(N, V, C)
    t = tgt.double().flatten()[:N * C * V].view(N, C, V).permute(0, 2, 1)
    if 'swap_C_cpad' in mut:    # rec and tgt indexed with the pitch cpad instead of C
        r = rec.double().flatten()[:N * V * cpad].view(N, V, cpad)[..., :C]
        t = tgt.double().flatten()[:N * cpad * V].view(N, cpad, V)[:, :C].permute(0, 2, 1)
    numel = N * V if 'coef_NV' in mut else N * C * V
    g = 1.0 if (gs is None or 'no_gscale' in mut) else gs
    ref = torch.zeros(N, V, cpad, dtype=F64T, device=rec.device)
    ref[..., :C] = (2.0 * g / numel) * (r - t)
    return ref, SLACK * (U + gam(2)) * ref.abs()


def test_bound_rejects_mse_mistakes():
    N, C, V, cpad = 2, 3, 37, 64
    rec = _rand((N * V * cpad,), 1100, dtype=F32T, device='cpu')     # room for the mistaken pitch
    tgt = _rand((N * cpad * V,), 1101, dtype=F32T, device='cpu')
    gs = f32(0.37)
    ref, tol = mse_bwd_expect(rec[:N * V * C], tgt[:N * C * V], gs, N, C, V, cpad)
    check('exact', ref.to(BF16), ref, tol)
    for mut in ('coef_NV', 'no_gscale', 'swap_C_cpad'):
        bad, _ = mse_bwd_expect(rec, tgt, gs, N, C, V, cpad, (mut,))
        _rejects(lambda: check(mut, bad.to(BF16), ref, tol))
    d = rec[:N * V * C].double().view(N, V, C).permute(0, 2, 1) - tgt[:N * C * V].double().view(N, C, V)
    s, tol = mse_fwd_expect(rec[:N * V * C], tgt[:N * C * V], N, C, V, 0.75, 132)
    s = float(s)
    check('fwd exact', torch.tensor(f32(s)), torch.tensor(s), tol)
    _rejects(lambda: check('fwd init dropped', torch.tensor(f32(s - 0.75)), torch.tensor(s), tol))
    _rejects(lambda: check('fwd last term dropped', torch.tensor(f32(s - float(d[-1, -1, -1] ** 2))),
                           torch.tensor(s), tol))


MSE_SHAPES = [(1, 1, 1), (3, 3, 1001), (8, 3, 16 * 64 * 64)]


@GPU
@pytest.mark.parametrize('N,C,V', MSE_SHAPES)
def test_mse(N, C, V):
    seed = 1200 + N + C
    rec, tgt = _rand((N, V, C), seed, dtype=F32T), _rand((N, C, V), seed + 1, 0.7, F32T)
    init = 0.75
    loss = Guarded((1,), F32T, init=torch.tensor([init]))
    _call('og_mse_fwd', rec.data_ptr(), tgt.data_ptr(), N, C, V, loss.ptr())
    torch.cuda.synchronize()
    loss.check_guard('loss_sum')
    check('loss_sum', loss.t[0], *mse_fwd_expect(rec, tgt, N, C, V, init, num_sms()))
    gsd = torch.tensor([0.37], dtype=F32T, device=DEV)
    for cpad in sorted({C, 8, 64}):
        for gs in (None, gsd):
            drec = Guarded((N, V, cpad), BF16)
            _call('og_mse_bwd', rec.data_ptr(), tgt.data_ptr(), None if gs is None else gs.data_ptr(), N, C, cpad, V,
                  drec.ptr())
            torch.cuda.synchronize()
            drec.check_guard('drec')
            ref, tol = mse_bwd_expect(rec, tgt, None if gs is None else f32(0.37), N, C, V, cpad)
            check(f'drec cpad={cpad} gs={gs is not None}', drec.t, ref, tol)
            assert bool((drec.t[..., C:].contiguous().view(torch.int16) == 0).all()), 'pad columns not +0'


@GPU
@pytest.mark.parametrize('n', [8, 8008, 2 ** 24])
def test_sqdiff_sum(n):
    """out = init + sum (a - b)^2. A term: the fp32 difference (1), its square in an fma (1), 8 fmas per iteration of
    its thread, 5 warp shuffles and one atomic per warp onto init."""
    a, b = _rand((n,), 1300 + n % 997), _rand((n,), 1301 + n % 997, 0.5)
    init = 2.5
    out = Guarded((1,), F32T, init=torch.tensor([init]))
    _call('og_sqdiff_sum', a.data_ptr(), b.data_ptr(), n, out.ptr())
    torch.cuda.synchronize()
    out.check_guard('out')
    d = a.double() - b.double()
    s = float((d * d).sum())
    blocks = ew_blocks(n // 8, num_sms())
    depth = 2 + 8 * cdiv(n // 8, blocks * 256) + 5 + blocks * 8
    check('sqdiff_sum', out.t[0], torch.tensor(init + s), gam(depth) * (init + s))


# ------------------------------------------------------------------------------------------------------------------
# blur pooling
# ------------------------------------------------------------------------------------------------------------------
def blur_weight(kt, k, mut=()):
    pas = lambda n: torch.tensor([math.comb(n - 1, i) for i in range(n)], dtype=F64T)
    w = pas(kt)[:, None, None] * pas(k)[None, :, None] * pas(k)[None, None, :]
    norm = w.sum() / (pas(kt).sum() if 'norm_2d' in mut else 1.0)
    return w / norm


def blur_fwd_ref(s, kt, k, stride, pad_t, pad, mut=()):
    """s: [N, T, H, W] float64 channel sums -> [N, To, Ho, Wo]: F.conv3d with the normalised Pascal kernel."""
    w = blur_weight(kt, k, mut)[None, None]
    x = s[:, None]
    if 'front_pad' in mut:      # all padding before the data, none after
        x = F.pad(x, (2 * pad, 0, 2 * pad, 0, 2 * pad_t, 0))
        return F.conv3d(x, w, stride=stride)[:, 0]
    return F.conv3d(x, w, stride=stride, padding=(pad_t, pad, pad))[:, 0]


def blur_bwd_ref(g, in_shape, kt, k, stride, pad_t, pad, mut=()):
    """g: [N, To, Ho, Wo] float64 -> the adjoint [N, T, H, W] by autograd. 'not_transposed' applies the forward stencil
    h + tap - pad instead of the adjoint h + pad - tap (index arithmetic as in og_blur3d_bwd_kernel)."""
    if 'not_transposed' in mut:
        N, T, H, W = in_shape
        w = blur_weight(kt, k)
        To, Ho, Wo = g.shape[1:]
        out = torch.zeros(in_shape, dtype=F64T)
        for t in range(T):
            for h in range(H):
                for x in range(W):
                    acc = torch.zeros(N, dtype=F64T)
                    for it in range(kt):
                        for ih in range(k):
                            for iw in range(k):
                                tn, hn, wn = t - pad_t + it, h - pad + ih, x - pad + iw
                                ok = all(v >= 0 and v % s == 0 and v // s < e for v, s, e in
                                         ((tn, stride[0], To), (hn, stride[1], Ho), (wn, stride[2], Wo)))
                                if ok:
                                    acc += w[it, ih, iw] * g[:, tn // stride[0], hn // stride[1], wn // stride[2]]
                    out[:, t, h, x] = acc
        return out
    s = torch.zeros(in_shape, dtype=F64T, device=g.device, requires_grad=True)
    y = blur_fwd_ref(s, kt, k, stride, pad_t, pad, mut)
    return torch.autograd.grad(y, s, g)[0]


def blur_expect(x, c_out, kt, k, stride, pad_t, pad, backward, in_shape=None, mut=()):
    """Reference and bound of either direction, broadcast to c_out channels. x: [N, ..., C_in_of_this_pass] bf16.
    Rounding points: the fp32 channel sum (ceil(C / 32) per lane + 5 shuffles), the fp32 stencil (one product and one
    add per tap; the Pascal weights and the power-of-two norm are exact), the bf16 store."""
    xs, xa = x.double().sum(-1), x.double().abs().sum(-1)
    if backward:
        ref = blur_bwd_ref(xs, in_shape, kt, k, stride, pad_t, pad, mut)
        mag = blur_bwd_ref(xa, in_shape, kt, k, stride, pad_t, pad)
    else:
        ref, mag = blur_fwd_ref(xs, kt, k, stride, pad_t, pad, mut), blur_fwd_ref(xa, kt, k, stride, pad_t, pad)
    depth = cdiv(x.shape[-1], 32) + 5 + kt * k * k + 1
    ref, mag = ref[..., None].expand(*ref.shape, c_out), mag[..., None].expand(*mag.shape, c_out)
    return ref, U * ref.abs() + SLACK * gam(depth) * mag


def test_bound_rejects_blur_mistakes():
    N, T, H, W, cin, cout = 2, 3, 6, 5, 8, 8
    # 3-D k = 3: a norm missing the time dimension, and all padding at the front
    x = _rand((N, T, H, W, cin), 1400, device='cpu')
    ex = blur_expect(x, cout, 3, 3, (1, 2, 2), 1, 1, False)
    check('fwd exact', ex[0].to(BF16), *ex)
    for mut in ('norm_2d', 'front_pad'):
        bad = blur_expect(x, cout, 3, 3, (1, 2, 2), 1, 1, False, mut=(mut,))[0]
        _rejects(lambda: check(mut, bad.to(BF16), *ex))
    # 2-D k = 4, stride 2, pad 1 (2 pad != k - 1, so the stencil is not its own transpose)
    st, k, pad = (1, 2, 2), 4, 1
    Ho, Wo = (H + 2 * pad - k) // 2 + 1, (W + 2 * pad - k) // 2 + 1
    dy = _rand((N, 1, Ho, Wo, cout), 1401, device='cpu')
    ex = blur_expect(dy, cin, 1, k, st, 0, pad, True, (N, 1, H, W))
    check('bwd exact', ex[0].to(BF16), *ex)
    loops = blur_expect(dy, cin, 1, k, st, 0, pad, True, (N, 1, H, W), mut=('not_transposed',))[0]
    _rejects(lambda: check('not transposed', loops.to(BF16), *ex))
    # the loop form with the adjoint indices is the autograd reference (pins the mutation to one index change)
    g = dy.double().sum(-1)
    w = blur_weight(1, k)
    sample = sum(w[0, ih, iw] * g[0, 0, (2 + pad - ih) // 2, (3 + pad - iw) // 2]
                 for ih in range(k) for iw in range(k)
                 if (2 + pad - ih) % 2 == 0 and (3 + pad - iw) % 2 == 0 and 0 <= (2 + pad - ih) // 2 < Ho
                 and 0 <= (3 + pad - iw) // 2 < Wo)
    assert abs(float(ex[0][0, 0, 2, 3, 0]) - float(sample)) < 1e-12


BLUR3D_CASES = [
    # (k, stride, (T, H, W), cin, cout)
    (1, (2, 2, 2), (3, 5, 7), 8, 8),
    (1, (2, 4, 4), (3, 9, 7), 64, 128),
    (3, (1, 1, 1), (1, 7, 9), 64, 128),
    (3, (2, 2, 2), (4, 9, 11), 128, 8),
    (3, (2, 4, 4), (5, 9, 13), 8, 8),          # stride > k: input voxels that no tap reaches get exactly 0
    (5, (1, 2, 2), (3, 3, 9), 8, 8),           # H < k
    (5, (3, 3, 3), (5, 11, 13), 64, 128),
    (7, (1, 1, 1), (1, 5, 9), 128, 8),         # T = 1, H < k
    (7, (2, 2, 2), (3, 7, 5), 8, 8),
]


def blur_run(dims, N, T, H, W, cin, cout, k, stride, pad, seed):
    kt, pad_t = (k, pad) if dims == 3 else (1, 0)
    st, sh, sw = stride
    To, Ho, Wo = (T + 2 * pad_t - kt) // st + 1, (H + 2 * pad - k) // sh + 1, (W + 2 * pad - k) // sw + 1
    x = _rand((N, T, H, W, cin), seed)
    dy = _rand((N, To, Ho, Wo, cout), seed + 1)
    y, dx = Guarded((N, To, Ho, Wo, cout), BF16), Guarded((N, T, H, W, cin), BF16)
    for bwd, src, dst, scratch_n in ((0, x, y, N * T * H * W), (1, dy, dx, N * To * Ho * Wo)):
        scratch = torch.empty(scratch_n, dtype=F32T, device=DEV)
        if dims == 3:
            _call('og_blurpool3d', src.data_ptr(), dst.ptr(), scratch.data_ptr(), bwd, N, T, H, W, cin, cout, k, st, sh,
                  sw)
        else:
            _call('og_blurpool2d', src.data_ptr(), dst.ptr(), scratch.data_ptr(), bwd, N, H, W, cin, cout, k, sh, sw,
                  pad)
    torch.cuda.synchronize()
    y.check_guard('y')
    dx.check_guard('dx')
    xc, dyc = x.cpu(), dy.cpu()
    check('y', y.t.cpu(), *blur_expect(xc, cout, kt, k, stride, pad_t, pad, False))
    ex = blur_expect(dyc, cin, kt, k, stride, pad_t, pad, True, (N, T, H, W))
    check('dx', dx.t.cpu(), *ex)
    return ex[0]


@GPU
@pytest.mark.parametrize('k,stride,thw,cin,cout', BLUR3D_CASES)
def test_blurpool3d(k, stride, thw, cin, cout):
    dx_ref = blur_run(3, 2, *thw, cin, cout, k, stride, (k - 1) // 2, 1500 + k + sum(thw))
    if any(s > k for s in stride):
        assert bool((dx_ref == 0).any())


@GPU
@pytest.mark.parametrize('k', [2, 3, 4, 5])
def test_blurpool2d(k):
    """stride 1, 2, 3 with pad = (k - 1) // stride (as BlurPooling2d uses) and pad = 0."""
    for s in (1, 2, 3):
        for pad in sorted({(k - 1) // s, 0}):
            blur_run(2, 2, 1, 9, 7, 16, 8, k, (1, s, s), pad, 1600 + 10 * k + s)


# ------------------------------------------------------------------------------------------------------------------
# AdamW
# ------------------------------------------------------------------------------------------------------------------
HYPER = {   # lr, beta1, beta2, eps, weight decay: the fp32 values the kernel receives
    'default': tuple(f32(h) for h in (1e-3, 0.9, 0.999, 1e-8, 1e-2)),
    'aggressive': tuple(f32(h) for h in (0.1, 0.5, 0.9, 1e-3, 0.1)),
}
STEPS = (1, 2, 10, 1000)
GS = f32(0.37)


def adam_exact(p, m, v, g, t, hp, gs=None, mut=()):
    """One torch.optim.AdamW step in float64 (decoupled decay, bias corrections at step t)."""
    lr, b1, b2, eps, wd = hp
    if gs is not None and 'no_gscale' not in mut:
        g = g * gs
    tc = t - 1 if 't_minus_1' in mut else t
    bc1, bc2sq = 1 - b1 ** tc, 1 - b2 ** tc
    if 'l2' in mut:
        g = g + wd * p
    elif 'decay_after' not in mut:
        p = p * (1 - lr * wd)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    if 'eps_inside' in mut:
        den = torch.sqrt(v / bc2sq + eps)
    elif 'bc2_no_sqrt' in mut:
        den = v.sqrt() / bc2sq + eps
    else:
        den = v.sqrt() / math.sqrt(bc2sq) + eps
    p = p - (lr / bc1 if bc1 else math.inf) * (m / den)      # bc1 = 0 only for 't_minus_1' at t = 1
    if 'decay_after' in mut:
        p = p * (1 - lr * wd)
    return p, m, v


def adam_bound(p, m, v, g, ep, em, ev, t, hp, gs, dev):
    """Bounds on |kernel - reference| of (p, m, v) after one step, given those before it. (p, m, v) is the float64
    reference state before the step. Every fp32 operation adds F32 times its result's magnitude; the bias corrections
    carry the host's rounding of a float64 value, or on the device powf's POWF_ULP ulps amplified by
    beta^t / (1 - beta^t), the fp32 subtraction and sqrtf."""
    lr, b1, b2, eps, wd = hp
    gg = g if gs is None else g * gs
    eg = 0.0 if gs is None else F32 * gg.abs()
    if dev:
        rb1 = (POWF_ULP * F32 * b1 ** t + 2.0 ** -140) / (1 - b1 ** t) + F32
        rb2 = 0.5 * ((POWF_ULP * F32 * b2 ** t + 2.0 ** -140) / (1 - b2 ** t) + F32) + F32
    else:
        rb1 = rb2 = F32
    dec = 1 - lr * wd
    p1 = p * dec
    ep1 = dec * ep + (p.abs() + ep) * F32 * (lr * wd + dec) + F32 * p1.abs()
    A, B = b1 * m.abs(), (1 - b1) * gg.abs()
    m1 = b1 * m + (1 - b1) * gg
    em1 = b1 * em + (1 - b1) * eg + F32 * 2 * (A + B)
    C, D = b2 * v, (1 - b2) * gg * gg
    v1 = C + D
    ev1 = b2 * ev + (1 - b2) * (2 * gg.abs() * eg + eg * eg) + F32 * (2 * C + 3 * D)
    bc1, bc2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
    sq = v1.sqrt()
    esq = torch.minimum(ev1.sqrt(), ev1 / sq.clamp_min(1e-300)) + F32 * (sq + ev1.sqrt())
    q = sq / bc2
    eq = esq / bc2 + (q + esq / bc2) * (rb2 + F32)
    den = q + eps
    eden = eq + F32 * den
    r = m1 / den
    er = (em1 + r.abs() * eden) / (den - eden).clamp_min(eps / 2) + F32 * (r.abs() + em1 / den)
    c = lr / bc1
    step = c * r
    estep = c * er + c * (r.abs() + er) * (rb1 + 2 * F32)
    p2 = p1 - step
    ep2 = ep1 + estep + F32 * (p1.abs() + ep1 + step.abs() + estep)
    return SLACK * ep2, SLACK * em1, SLACK * ev1


def adam_fp32(p, m, v, g, t, hp, gs=None):
    """The kernel's scalar loop in fp32 on the CPU, host-side bias corrections: a correct kernel."""
    lr, b1, b2, eps, wd = (torch.tensor(h, dtype=F32T) for h in hp)
    bc1 = torch.tensor(1 - float(b1) ** t, dtype=F32T)
    bc2 = torch.tensor(math.sqrt(1 - float(b2) ** t), dtype=F32T)
    if gs is not None:
        g = g * torch.tensor(gs, dtype=F32T)
    p = p * (1 - lr * wd)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    p = p - (lr / bc1) * (m / (torch.sqrt(v) / bc2 + eps))
    return p, m, v


def _grad_scale(n, hp, seed, device):
    """Per-element gradient magnitudes, log-uniform down to where sqrt(v_hat) is about eps."""
    lo = math.log10(hp[3]) - 0.5
    return 10.0 ** (torch.rand(n, generator=_gen(seed, device), device=device, dtype=F64T) * -lo + lo)


def test_bound_rejects_adamw_mistakes():
    n = 4096
    for hname, hp in HYPER.items():
        p0 = _rand((n,), 1700, 0.1, F32T, 'cpu')
        scale = _grad_scale(n, hp, 1701, 'cpu')
        grads = [(_rand((n,), 1702 + i, 1.0, F64T, 'cpu') * scale).float() for i in range(len(STEPS))]

        def run(mut, gs):
            """Checks the fp32 emulation (mut = None) or a float64 mistake rounded to fp32 against the bound."""
            P, M, Vv = p0.double(), torch.zeros(n, dtype=F64T), torch.zeros(n, dtype=F64T)
            ep = em = ev = torch.zeros(n, dtype=F64T)
            kp, km, kv = p0.clone(), torch.zeros(n), torch.zeros(n)
            for t, g in zip(STEPS, grads):
                if mut is None:
                    kp, km, kv = adam_fp32(kp, km, kv, g, t, hp, gs)
                else:
                    kp, km, kv = (a.float() for a in adam_exact(kp.double(), km.double(), kv.double(), g.double(), t,
                                                                hp, gs, (mut,)))
                ep, em, ev = adam_bound(P, M, Vv, g.double(), ep, em, ev, t, hp, gs, False)
                P, M, Vv = adam_exact(P, M, Vv, g.double(), t, hp, gs)
                check(f'{hname} {mut} p t={t}', kp, P, ep)
                check(f'{hname} {mut} m t={t}', km, M, em)
                check(f'{hname} {mut} v t={t}', kv, Vv, ev)
        run(None, None)
        run(None, GS)
        muts = ['eps_inside', 'bc2_no_sqrt', 'l2', 't_minus_1', 'no_gscale']
        if hname == 'aggressive':
            muts.append('decay_after')   # at lr = 1e-3, wd = 1e-2 the difference (lr^2 wd) is below fp32's resolution
        for mut in muts:
            _rejects(lambda: run(mut, GS))


ADAM_SPEC = [
    # name, n, p offset (floats), gradient given, bf16 destination (row_len, dst_ld, column offset) or None
    ('big', 1100 * 2048 + 777, 0, True, (512, 512, 0)),   # vector chunks, a scalar tail, > 8 chunks per SM
    ('p_off1', 5000, 1, True, None),                       # p one float off 16-byte alignment: scalar
    ('row18', 6 * 2048, 0, True, (18, 64, 0)),             # row_len % 4 != 0 (the padded stem form): scalar
    ('no_grad', 4096 + 100, 0, False, (100, 100, 0)),      # g NULL: p, m, v untouched, bf16 copy refreshed
    ('no_bf16', 4096, 0, True, None),                      # vector, no bf16 copy
    ('pitched', 64 * 64, 0, True, (64, 96, 16)),           # dst_ld > row_len, segment at column 16: vector
    ('ld_odd', 2 * 2048, 0, True, (64, 66, 0)),            # dst_ld % 4 != 0: scalar
    ('bf16_off', 2048, 0, True, (64, 128, 1)),             # p_bf16 2 bytes off 8-byte alignment: scalar
]
ADAM_VEC = {'big', 'no_bf16', 'pitched'}                 # entries with vector chunks; every entry but these is scalar


def adam_vec(base, n, p, g, m, v, pb, row_len, dst_ld):
    """Mirror of og_adamw_kernel's vector predicate for the chunk starting at element `base` (byte addresses)."""
    return (base + 2048 <= n and bool(g) and all((a + 4 * base) % 16 == 0 for a in (p, g, m, v))
            and row_len % 4 == 0 and (not pb or (pb % 8 == 0 and dst_ld % 4 == 0)))


def test_adamw_vector_predicate_mirror():
    a = 1 << 20      # 16-byte aligned base address
    assert adam_vec(0, 4096, a, a, a, a, 0, 4, 4) and adam_vec(2048, 4096, a, a, a, a, a, 64, 96)
    assert not adam_vec(0, 4096, a, a, a, a, 0, 1, 1)     # row_len 1, as FusedAdamW passes without a bf16 target
    assert not adam_vec(2048, 4095, a, a, a, a, 0, 1, 1)                  # partial chunk
    assert not adam_vec(0, 4096, a + 4, a, a, a, 0, 1, 1)                 # p off alignment
    assert not adam_vec(0, 4096, a, 0, a, a, a, 64, 64)                   # no gradient
    assert not adam_vec(0, 4096, a, a, a, a, a, 18, 64)                   # row_len % 4
    assert not adam_vec(0, 4096, a, a, a, a, a, 64, 66)                   # dst_ld % 4
    assert not adam_vec(0, 4096, a, a, a, a, a + 2, 64, 64)               # p_bf16 off 8-byte alignment
    assert adam_vec(0, 4096, a, a, a, a, a + 8, 64, 64)


def adam_setup(hp, seed):
    ents = []
    for i, (name, n, poff, grad, dst) in enumerate(ADAM_SPEC):
        e = {'name': name, 'n': n, 'grad': grad, 'dst': dst,
             'p': Guarded((n,), F32T, init=_rand((n,), seed + 10 * i, 0.1, F32T), offset=poff),
             'm': Guarded((n,), F32T, init=torch.zeros(n)), 'v': Guarded((n,), F32T, init=torch.zeros(n)),
             'scale': _grad_scale(n, hp, seed + 10 * i + 1, DEV), 'pb': 0}
        if dst:
            row_len, ld, col = dst
            e['D'] = Guarded((cdiv(n, row_len), ld), BF16)
            e['pb'] = e['D'].ptr() + 2 * col
        ents.append(e)
    nch = [cdiv(e['n'], 2048) for e in ents]
    ct = torch.repeat_interleave(torch.arange(len(ents)), torch.tensor(nch))
    ci = torch.cat([torch.arange(c) for c in nch])
    perm = torch.randperm(ct.numel(), generator=torch.Generator().manual_seed(seed))
    return ents, ct[perm].int(), ci[perm].int()


def adam_table(ents, grads):
    from open_genie_b200 import _lib
    tab = (_lib.og_adamw_tensor * len(ents))()
    for t, e in zip(tab, ents):
        t.p, t.m, t.v = e['p'].ptr(), e['m'].ptr(), e['v'].ptr()
        t.g = grads[e['name']].data_ptr() if e['grad'] else None
        t.p_bf16 = e['pb'] or None
        t.n = e['n']
        t.row_len, t.dst_ld = (e['dst'][0], e['dst'][1]) if e['dst'] else (4, 4)
    return torch.frombuffer(bytearray(bytes(tab)), dtype=torch.uint8).to(DEV)


def _bf16_dst_expect(e):
    """The whole destination buffer as it must be: NaN bits everywhere except bf16(p) at each element's position."""
    row_len, ld, col = e['dst']
    want = torch.full_like(e['D'].buf.view(torch.int16), Guarded.BITS[BF16][1])
    i = torch.arange(e['n'], device=DEV)
    want[(i // row_len) * ld + col + i % row_len] = e['p'].t.to(BF16).view(torch.int16)
    return want


@GPU
@pytest.mark.parametrize('hyper', sorted(HYPER))
@pytest.mark.parametrize('mode', ['host', 'device'])
def test_adamw_step(mode, hyper):
    """One launch per step over a shuffled chunk table with every kind of entry, at t = 1, 2, 10, 1000. 'device' reads
    the step count, the learning rate and a gradient scale of 0.37 from device memory; the host arguments then carry
    decoys (step 999, lr 0.5) that must be ignored."""
    hp = HYPER[hyper]
    dev = mode == 'device'
    ents, ct, ci = adam_setup(hp, 1800 + 7 * len(hyper) + dev)
    nchunks = ct.numel()
    assert nchunks > 8 * num_sms()
    ct_d, ci_d = ct.to(DEV), ci.to(DEV)      # held for the launches: a temporary's memory could be reused at once
    by_name = {e['name']: e for e in ents}
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    lr_dev = torch.tensor([hp[0]], dtype=F32T, device=DEV)
    gs_dev = torch.tensor([GS], dtype=F32T, device=DEV)
    gs = GS if dev else None
    ref = {e['name']: dict(p=e['p'].t.double(), m=torch.zeros(e['n'], dtype=F64T, device=DEV),
                           v=torch.zeros(e['n'], dtype=F64T, device=DEV), ep=0.0, em=0.0, ev=0.0,
                           bits=[e[k].t.clone() for k in 'pmv']) for e in ents}
    for step_i, t in enumerate(STEPS):
        grads = {e['name']: (_rand((e['n'],), 1900 + 31 * step_i + j, 1.0, F64T) * e['scale']).float()
                 for j, e in enumerate(ents)}
        if step_i == 0:   # the vector predicate, mirrored on the real addresses: which entries take which path
            vec = {}
            for c_t, c_i in zip(ct.tolist(), ci.tolist()):
                e = ents[c_t]
                g = grads[e['name']].data_ptr() if e['grad'] else 0
                rl, ld = (e['dst'][0], e['dst'][1]) if e['dst'] else (4, 4)
                vec.setdefault(e['name'], set()).add(adam_vec(c_i * 2048, e['n'], e['p'].ptr(), g, e['m'].ptr(),
                                                              e['v'].ptr(), e['pb'], rl, ld))
            assert {k for k, s in vec.items() if True in s} == ADAM_VEC, vec
            assert {k for k, s in vec.items() if False in s} == set(by_name) - {'no_bf16', 'pitched'}, vec
        table = adam_table(ents, grads)
        lr, b1, b2, eps, wd = hp
        if dev:
            step_dev.fill_(t)
            _call('og_adamw_step', table.data_ptr(), ct_d.data_ptr(), ci_d.data_ptr(), nchunks, 0.5, b1, b2, eps, wd,
                  999, step_dev.data_ptr(), lr_dev.data_ptr(), gs_dev.data_ptr())
        else:
            _call('og_adamw_step', table.data_ptr(), ct_d.data_ptr(), ci_d.data_ptr(), nchunks, lr, b1, b2, eps, wd, t,
                  None, None, None)
        torch.cuda.synchronize()
        for e in ents:
            name, r = e['name'], ref[e['name']]
            for k in 'pmv':
                e[k].check_guard(f'{name}.{k}')
            if e['grad']:
                g = grads[name].double()
                r['ep'], r['em'], r['ev'] = adam_bound(r['p'], r['m'], r['v'], g, r['ep'], r['em'], r['ev'], t, hp,
                                                       gs, dev)
                r['p'], r['m'], r['v'] = adam_exact(r['p'], r['m'], r['v'], g, t, hp, gs)
                for k in 'pmv':
                    check(f'{name}.{k} t={t}', e[k].t, r[k], r['e' + k])
            else:
                for k, b in zip('pmv', r['bits']):
                    check_bits(f'{name}.{k} (no gradient) t={t}', e[k].t, b)
            if e['dst']:
                got = e['D'].buf.view(torch.int16)
                want = _bf16_dst_expect(e)
                bad = got != want
                assert not bad.any(), f'{name}: {int(bad.sum())} bf16 destination elements wrong (first at flat ' \
                                      f'{int(torch.nonzero(bad)[0])})'


# ------------------------------------------------------------------------------------------------------------------
# FusedAdamW: each form of bf16 operand target
# ------------------------------------------------------------------------------------------------------------------
def _fused_steps(params_lr, opt, nsteps, seed):
    """Runs nsteps of `opt` with fresh gradients and checks every parameter and its moments against float64 AdamW
    (device-side bias corrections: FusedAdamW passes its step counter)."""
    ref = {id(p): dict(p=p.detach().reshape(-1).double(), m=torch.zeros(p.numel(), dtype=F64T, device=DEV),
                       v=torch.zeros(p.numel(), dtype=F64T, device=DEV), ep=0.0, em=0.0, ev=0.0) for p, _ in params_lr}
    for t in range(1, nsteps + 1):
        for i, (p, _) in enumerate(params_lr):
            p.grad = torch.randn_like(p) * 0.01 * (i + 1)
        opt.step()
        torch.cuda.synchronize()
        for i, (p, lr) in enumerate(params_lr):
            hp = (f32(lr),) + HYPER['default'][1:]
            r, g = ref[id(p)], p.grad.reshape(-1).double()
            r['ep'], r['em'], r['ev'] = adam_bound(r['p'], r['m'], r['v'], g, r['ep'], r['em'], r['ev'], t, hp, None,
                                                   True)
            r['p'], r['m'], r['v'] = adam_exact(r['p'], r['m'], r['v'], g, t, hp)
            st = opt.state[p]
            check(f'param {i} t={t}', p.detach().reshape(-1), r['p'], r['ep'])
            check(f'exp_avg {i} t={t}', st['exp_avg'].reshape(-1), r['m'], r['em'])
            check(f'exp_avg_sq {i} t={t}', st['exp_avg_sq'].reshape(-1), r['v'], r['ev'])


def _operand(conv):
    """[cout][taps * cin] bf16 rows of a conv weight in the packed operand's order (tap-major, channel-minor)."""
    w = conv.weight.detach()
    return w.permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1, w.shape[1])


@GPU
def test_fused_adamw_shortcut_block():
    """Main 3x3x3 conv with a fused 1x1x1 shortcut: after each step the packed operand is exactly the bf16 cast of
    [main | shortcut], and no other column changes."""
    from open_genie_b200.module.video import Conv3dParams
    from open_genie_b200.optim import FusedAdamW
    torch.manual_seed(2000)
    main, sc = Conv3dParams(64, 64, (3, 3, 3)).to(DEV), Conv3dParams(32, 64, (1, 1, 1)).to(DEV)
    main.fuse_shortcut(sc)
    params = [main.weight, main.bias, sc.weight, sc.bias]
    opt = FusedAdamW(params, lr=1e-3)
    _fused_steps([(p, 1e-3) for p in params], opt, 2, 2001)
    packed = main.packed()
    assert packed.shape == (64, 27 * 64 + 32)
    want = torch.cat([_operand(main).reshape(64, -1), _operand(sc).reshape(64, -1)], 1).to(BF16)
    check_bits('packed [main | shortcut]', packed, want)


@GPU
@pytest.mark.parametrize('cin', [3, 18])
def test_fused_adamw_padded_stem(cin):
    """Stem conv with cin padded to 64 per tap: the cin columns of each tap are bf16(weight), the pad columns stay +0."""
    from open_genie_b200.module.video import Conv3dParams
    from open_genie_b200.optim import FusedAdamW
    torch.manual_seed(2100 + cin)
    conv = Conv3dParams(cin, 64, (3, 3, 3)).to(DEV)
    assert conv.geom.padded and conv.geom.cin_pad == 64
    opt = FusedAdamW([conv.weight, conv.bias], lr=1e-3)
    _fused_steps([(conv.weight, 1e-3), (conv.bias, 1e-3)], opt, 2, 2101)
    packed = conv.packed().view(64, 27, 64)
    check_bits('weight columns', packed[..., :cin], _operand(conv).to(BF16))
    assert bool((packed[..., cin:].contiguous().view(torch.int16) == 0).all()), 'pad columns changed'


@GPU
def test_fused_adamw_two_groups():
    """Two parameter groups with different learning rates: one launch each, each against its own reference."""
    from open_genie_b200.module.video import Conv3dParams
    from open_genie_b200.optim import FusedAdamW
    torch.manual_seed(2200)
    a, b = Conv3dParams(64, 64, (1, 1, 1)).to(DEV), Conv3dParams(64, 128, (1, 3, 3)).to(DEV)
    opt = FusedAdamW([{'params': [a.weight, a.bias], 'lr': 1e-3}, {'params': [b.weight, b.bias], 'lr': 0.05}])
    _fused_steps([(a.weight, 1e-3), (a.bias, 1e-3), (b.weight, 0.05), (b.bias, 0.05)], opt, 3, 2201)
    for conv in (a, b):
        check_bits('packed', conv.packed(), _operand(conv).reshape(conv.out_channels, -1).to(BF16))


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation (host buffers, no launch)
# ------------------------------------------------------------------------------------------------------------------
def test_layout_argument_validation_returns_status_codes():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    p = (ctypes.addressof(buf) + 15) & ~15          # 16-byte aligned
    q = p + 2                                       # 2-byte aligned only

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error())
    # og_colsum with rows <= 0 (used to divide by zero on the host)
    bad(lib.og_colsum(p, 0, 8, 8, p, None), b'colsum: bad arguments')
    bad(lib.og_colsum(p, -3, 8, 8, p, None), b'colsum: bad arguments')
    bad(lib.og_colsum(p, 16, 8, 4, p, None), b'colsum: bad arguments')
    # 16-byte vector accesses need 16-byte aligned pointers
    for a, b_, o in ((q, p, p), (p, q, p), (p, p, q)):
        bad(lib.og_sub_rows(a, b_, o, 8, None), b'16-byte aligned')
    for x, y in ((q, p), (p, q)):
        bad(lib.og_maxpool2x2(x, y, 1, 2, 2, 8, None), b'16-byte aligned')
        bad(lib.og_sqdiff_sum(x, y, 8, p, None), b'16-byte aligned')
    for bwd in (0, 1):
        bad(lib.og_blurpool3d(p, q, p, bwd, 1, 2, 4, 4, 8, 8, 3, 1, 1, 1, None), b'16-byte aligned')
        bad(lib.og_blurpool2d(p, q, p, bwd, 1, 4, 4, 8, 8, 3, 1, 1, 1, None), b'16-byte aligned')
    # blur pooling: non-positive extents, and a padded extent smaller than the kernel (H = 2, k = 5, pad = 1, s = 3
    # used to give one output row where F.conv2d raises)
    for N, T, H, W in ((0, 1, 4, 4), (1, 0, 4, 4), (1, 1, 0, 4), (1, 1, 4, -1)):
        bad(lib.og_blurpool3d(p, p, p, 0, N, T, H, W, 8, 8, 3, 1, 1, 1, None), b'bad extents')
    bad(lib.og_blurpool2d(p, p, p, 1, -1, 4, 4, 8, 8, 3, 1, 1, 1, None), b'bad extents')
    bad(lib.og_blurpool2d(p, p, p, 0, 1, 2, 8, 8, 8, 5, 3, 3, 1, None), b'smaller than the kernel')
    bad(lib.og_blurpool2d(p, p, p, 1, 1, 8, 2, 8, 8, 5, 3, 3, 1, None), b'smaller than the kernel')
    bad(lib.og_blurpool2d(p, p, p, 0, 1, 3, 3, 8, 8, 4, 1, 1, 0, None), b'smaller than the kernel')
    # pixel shuffle: non-positive extents
    for N, T, H, W in ((0, 1, 1, 1), (1, 0, 1, 1), (1, 1, -2, 1), (1, 1, 1, 0)):
        bad(lib.og_pixel_shuffle3d(p, p, 0, N, T, H, W, 8, 2, 2, 2, None), b'bad extents')
    # the checks that already existed
    bad(lib.og_pixel_shuffle3d(p, p, 0, 1, 1, 1, 1, 0, 2, 2, 2, None), b'bad shape')
    bad(lib.og_pixel_shuffle3d(p, p, 0, 1, 1, 1, 1, 8, 2, 0, 2, None), b'bad shape')
    bad(lib.og_blurpool3d(p, p, p, 0, 1, 2, 4, 4, 12, 8, 3, 1, 1, 1, None), b'C % 8 == 0')
    bad(lib.og_blurpool3d(p, p, p, 0, 1, 2, 4, 4, 8, 8, 9, 1, 1, 1, None), b'k <= 7')
    bad(lib.og_blurpool3d(p, p, p, 0, 1, 2, 4, 4, 8, 8, 4, 1, 1, 1, None), b'odd kernel sizes')
    bad(lib.og_blurpool2d(p, p, p, 0, 1, 4, 4, 8, 8, 3, 0, 1, 1, None), b'bad stride')
    bad(lib.og_maxpool2x2(p, p, 1, 2, 2, 12, None), b'multiple of 8')
    bad(lib.og_sub_rows(p, p, p, 12, None), b'multiple of 8')
    bad(lib.og_sqdiff_sum(p, p, 12, p, None), b'n % 8 == 0')
    bad(lib.og_mse_bwd(p, p, None, 1, 3, 2, 16, p, None), b'mse_bwd: bad arguments')


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
PIN_CASES = [('pixel_shuffle', c) for c in sorted(PS_CASES) if 'grid_stride' not in c] + \
    [('colsum', c) for c in sorted(COLSUM_CASES) if c != 'vec_524288x128']


@GPU
@pytest.mark.parametrize('kind,case', PIN_CASES)
def test_dispatch_kernel_names(kind, case):
    """The shapes and offsets above reach the kernel the plan mirrors say they do."""
    if kind == 'pixel_shuffle':
        names = _kernels_run(lambda: pixel_shuffle_run(case, 2300))
        want = ps_plan(*PS_CASES[case])[0]
        others = [k for k in PS_KERNELS if k != want]
    else:
        names = _kernels_run(lambda: colsum_run(case, 2400))
        want = colsum_plan(*COLSUM_CASES[case], num_sms())[0]
        others = [k for k in ('og_colsum_vec_kernel', 'og_colsum_kernel(') if k != want]
    launched = sorted(set(n for n in names if 'og_' in n))
    assert any(want in n for n in names), (case, want, launched)
    for o in others:
        assert not any(o in n for n in names), (case, o, launched)
