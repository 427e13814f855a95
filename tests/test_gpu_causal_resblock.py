"""Causal video residual blocks and grouped blur pooling (genie/module/video.py:539-656, 487-537, 106-200).

- Kernel level: og_blurpool3d_grouped forward and backward against float64 on the same bf16 inputs, element by element
  in `Guarded` buffers, over groups, kernel sizes, strides, ragged extents and cout != cin; groups == 1 bit-identical
  to og_blurpool3d; argument checks returning status codes (CPU).
- Module level: every case of tests/golden/causal_resblock.pt (made by oracle/make_golden_causal.py from the unmodified
  reference) against the golden and against oracle.causal_oracle on bf16-rounded weights; state_dict keys and loading
  a reference-layout state dict; the fused causal block against its module-by-module composition; the convolution
  padding the fused block passes to og_conv3d_fwd; the refusals.
- Model level: the causal mini tokenizer's training loss and gradients against the golden, tokenize / decode shapes,
  and a GraphedTrainStep replay against the eager step.
- CPU: construction, keys, refusals, and the oracle against the golden.
"""
import ctypes
import math
import re

import pytest
import torch
import torch.nn.functional as F

from helpers import Guarded, bf16_round, det_weights, rel_l2, round_conv_weights
from oracle import causal_oracle as C
from oracle import genie_oracle as O

GPU = pytest.mark.gpu
DEV = 'cuda'
BF16, F32T, F64T = torch.bfloat16, torch.float32, torch.float64
GOLDEN = 'causal_resblock.pt'
BLOCKS = ('video_plain', 'video_causal_g2', 'video_leaky_down24', 'video_causal_g2_leaky_down24', 'causal_down12',
          'causal_down2', 'causal_k1')

# rounding model of test_gpu_layout_optim_paths.py: U is bf16's unit roundoff, F32 one fp32 ulp per operation
U = 2.0 ** -8
F32 = 2.0 ** -23
SLACK = 1.02


def _block(kw):
    from open_genie_b200.module.video import VideoResidualBlock
    return VideoResidualBlock(**kw)


def _oracle_block(kw):
    return lambda sd, x: C.video_residual_block(sd, '', x, kw.get('num_groups', 1), kw.get('downsample'),
                                                kw.get('use_causal', False), kw.get('act_fn', 'swish'))


def _case_module_and_oracle(tag, g):
    from open_genie_b200.module.discriminator import VideoDiscriminator
    from open_genie_b200.module.video import BlurPooling3d
    kw = g['kw']
    if tag == 'blur_g4':
        return BlurPooling3d(**kw), lambda sd, x: O.blur_pool3d(x, 3, 2, 2, kw['num_groups'], kw['out_channels'])
    if tag == 'video_disc_g2':
        return VideoDiscriminator(**kw), lambda sd, x: C.video_discriminator(sd, x, (64, 128, 256), (None, 2, 2),
                                                                             kw['num_groups'])
    return _block(kw), _oracle_block(kw)


def _ill_conditioned(m, k):
    """The first conv's bias gradient in a down-sampling block. Blur pooling makes the gradient at that conv's output
    equal over the channels of a group, and the GroupNorm after the pooling removes its mean over the group, so the
    bias gradient is a sum whose terms cancel: on the critic case it is 1/79 of the sum of their magnitudes, and
    rounding the weights to bf16 alone moves the fp32 reference by 13 %. It is not compared element by element."""
    if not re.search(r'main\.2\.(conv3d\.)?bias$', k):
        return False
    return getattr(m.get_submodule(k.split('main.2.')[0].rstrip('.')), 'has_down', False)


def _sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)]


# ------------------------------------------------------------------------------------------------------------------
# CPU: construction, keys, refusals, oracle against the golden
# ------------------------------------------------------------------------------------------------------------------
def test_state_dict_keys_equal_the_reference(golden):
    import open_genie_b200 as og
    g = golden(GOLDEN)
    for tag, case in g.items():
        if tag == 'tokenizer':
            m = og.VideoTokenizer(case['enc'], case['dec'], d_codebook=case['d_codebook'], gan_loss_weight=0,
                                  perc_loss_weight=0)
        else:
            m = _case_module_and_oracle(tag, case)[0]
        got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert got == case['keys'], (tag, set(got) ^ set(case['keys']))
    causal = g['video_causal_g2_leaky_down24']['keys']
    assert {'main.2.conv3d.weight', 'main.6.conv3d.bias', 'res.1.conv3d.weight', 'main.3.blur', 'res.0.blur'} <= set(causal)
    assert 'main.2.weight' in g['video_plain']['keys'] and 'res.1.weight' in g['video_plain']['keys']


def test_reference_layout_state_dict_loads_and_fuses_the_shortcut(golden):
    import copy
    g = golden(GOLDEN)['video_causal_g2']
    m = _block(g['kw'])
    sd = O.det_state_dict(g['keys'])
    m.load_state_dict(sd, strict=True)
    for k, v in sd.items():
        assert torch.equal(m.state_dict()[k], v), k
    assert m.main[6].conv3d._extra is m.res[1].conv3d
    c = copy.deepcopy(m)
    assert c.main[6].conv3d._extra is c.res[1].conv3d and c.res[1].conv3d._fused_into() is c.main[6].conv3d


def test_refusals():
    from open_genie_b200.module.discriminator import VideoDiscriminator
    from open_genie_b200.module.video import BlurPooling3d, CausalConv3d, VideoResidualBlock
    with pytest.raises(NotImplementedError, match='use_blur=False'):
        VideoResidualBlock(64, 128, downsample=2, use_blur=False, use_causal=True)
    with pytest.raises(NotImplementedError):
        VideoResidualBlock(64, 128, use_causal=True, pad_mode='reflect')
    with pytest.raises(NotImplementedError):
        VideoDiscriminator(inp_size=(8, 16, 16), use_causal=True)
    # the padding quirk: harmless only when (k - 1) // 2 is the same in all three dimensions
    for k in ((3, 5, 5), (1, 3, 3), (5, 3, 3)):
        with pytest.raises(NotImplementedError, match='reads the padding tuple'):
            VideoResidualBlock(64, use_causal=True, kernel_size=k)
    for k in (1, 3, 5, (3, 4, 4)):
        VideoResidualBlock(64, use_causal=True, kernel_size=k)
    # CausalConv3d: a padding that resolves to the default spatial pads, nothing else
    for pad in (None, 1, (1, 1), (None, 1), (1, 1, 1), (1, 1, 7)):
        CausalConv3d(8, 8, 3, padding=pad)
    CausalConv3d(8, 8, (3, 5, 1), padding=(2, 0))
    for pad in (0, 2, (1, 0), (0, 1, 1), (1,), 'same'):
        with pytest.raises(NotImplementedError):
            CausalConv3d(8, 8, 3, padding=pad)
    with pytest.raises(NotImplementedError):
        CausalConv3d(8, 8, 3, pad_mode='reflect')
    with pytest.raises(ValueError):
        BlurPooling3d(64, 3, out_channels=6, num_groups=4)
    VideoDiscriminator(inp_size=(8, 16, 16), num_groups=2)


def test_oracle_matches_golden(golden):
    """oracle.causal_oracle on the golden's closed-form weights and inputs reproduces the reference's samples."""
    g = golden(GOLDEN)
    for tag, case in g.items():
        if tag == 'tokenizer':
            continue
        sd = O.det_state_dict(case['keys'])
        sd = {k: v.requires_grad_(True) for k, v in sd.items()}
        x = O.det_uniform(f'causal.x.{tag}', case['shape']).requires_grad_(True)
        y = _case_module_and_oracle(tag, case)[1](sd, x)
        y.square().mean().backward()
        assert tuple(y.shape) == case['y_shape'], tag
        torch.testing.assert_close(_sample(f'causal.y.{tag}', y, 256), case['y'], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(_sample(f'causal.dx.{tag}', x.grad, 256), case['dx'], rtol=1e-4, atol=1e-8)
        for k in case['grad_names']:
            assert abs(sd[k].grad.norm().item() - case['grad_norm'][k]) <= 1e-4 * case['grad_norm'][k] + 1e-9, k
    t = g['tokenizer']
    sd = O.det_state_dict(t['keys'])
    video = O.det_uniform('causal.tokenizer.video', t['video_shape'])
    loss, (rec, ql), _, _ = C.tokenizer_forward(sd, t['enc'], t['dec'], video, t['d_codebook'])
    assert abs(loss.item() - t['loss']) <= 1e-4 * t['loss']
    assert abs(rec.item() - t['rec_loss']) <= 1e-4 * t['rec_loss']
    q, idxs = C.tokenizer_tokenize(sd, t['enc'], video, t['d_codebook'])
    assert torch.equal(idxs, t['idxs']) and tuple(q.shape) == t['quant_shape']


def test_grouped_blur_argument_validation_returns_status_codes():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    p = (ctypes.addressof(buf) + 15) & ~15
    q = p + 2

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error())
    f = lib.og_blurpool3d_grouped
    for bwd in (0, 1):
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 16, 16, 3, 3, 1, 1, 1, None), b'must divide')        # 3 does not divide 16
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 16, 16, 0, 3, 1, 1, 1, None), b'must divide')
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 16, 32, 4, 3, 1, 1, 1, None), b'(cin/groups) % 8')   # 4-channel input groups
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 32, 16, 4, 3, 1, 1, 1, None), b'(cout/groups) % 8')
        bad(f(None, p, p, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'null pointer')
        bad(f(p, None, p, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'null pointer')
        bad(f(p, p, None, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'null pointer')
        bad(f(q, p, p, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'x must be 16-byte aligned')
        bad(f(p, q, p, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'y must be 16-byte aligned')
        bad(f(p, p, q, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'scratch must be 4-byte aligned')
        bad(f(p, p, p, bwd, 0, 2, 4, 4, 16, 16, 2, 3, 1, 1, 1, None), b'bad extents')
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 16, 16, 2, 4, 1, 1, 1, None), b'odd kernel sizes')
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 16, 16, 2, 9, 1, 1, 1, None), b'k <= 7')
        bad(f(p, p, p, bwd, 1, 2, 4, 4, 16, 16, 2, 3, 0, 1, 1, None), b'bad stride')


# ------------------------------------------------------------------------------------------------------------------
# kernel level: og_blurpool3d_grouped against float64
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _rand(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV).to(BF16)


def _blur64(s, k, stride, pad, transpose_to=None):
    """s: [N, G, T, H, W] float64 -> the blur of each group (forward), or its adjoint onto `transpose_to` extents."""
    row = torch.tensor([math.comb(k - 1, i) for i in range(k)], dtype=F64T)
    w = row[:, None, None] * row[None, :, None] * row[None, None, :]
    w = (w / w.sum())[None, None].to(s.device)
    N, G = s.shape[:2]
    flat = s.reshape(N * G, 1, *s.shape[2:])
    if transpose_to is None:
        out = F.conv3d(flat, w, stride=stride, padding=pad)
    else:
        z = torch.zeros(N * G, 1, *transpose_to, dtype=F64T, device=s.device, requires_grad=True)
        out = torch.autograd.grad(F.conv3d(z, w, stride=stride, padding=pad), z, flat)[0]
    return out.reshape(N, G, *out.shape[2:])


def grouped_expect(x, G, c_out, k, stride, backward, in_thw=None):
    """Reference and per-element bound of either direction, broadcast over each group's c_out / G channels.
    x: [N, T, H, W, C] bf16 with C the channels summed in this pass. Rounding points: the fp32 group sum (C/G - 1
    adds in channel order), the fp32 stencil (one product and one add per tap; Pascal weights and the power-of-two
    norm are exact), the bf16 store."""
    N, C = x.shape[0], x.shape[-1]
    xs = x.double().reshape(*x.shape[:-1], G, C // G)
    s, a = xs.sum(-1).permute(0, 4, 1, 2, 3), xs.abs().sum(-1).permute(0, 4, 1, 2, 3)
    pad = (k - 1) // 2
    ref = _blur64(s, k, stride, pad, in_thw if backward else None)
    mag = _blur64(a, k, stride, pad, in_thw if backward else None)
    depth = C // G + k ** 3 + 1
    ref = ref.permute(0, 2, 3, 4, 1).repeat_interleave(c_out // G, dim=-1)
    mag = mag.permute(0, 2, 3, 4, 1).repeat_interleave(c_out // G, dim=-1)
    return ref, U * ref.abs() + SLACK * depth * F32 * mag


def _check(name, got, ref, tol):
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f'{name}: {int(bad.sum())}/{bad.numel()} outside the bound; first at flat {i}: got '
                             f'{got.flatten()[i].item():.9g} ref {ref.flatten()[i].item():.9g} bound '
                             f'{tol.flatten()[i].item():.3g}')


def grouped_run(N, T, H, W, cin, cout, G, k, stride, seed):
    st, sh, sw = stride
    pad = (k - 1) // 2
    To, Ho, Wo = (T + 2 * pad - k) // st + 1, (H + 2 * pad - k) // sh + 1, (W + 2 * pad - k) // sw + 1
    x = _rand((N, T, H, W, cin), seed)
    dy = _rand((N, To, Ho, Wo, cout), seed + 1)
    y, dx = Guarded((N, To, Ho, Wo, cout), BF16), Guarded((N, T, H, W, cin), BF16)
    for bwd, src, dst, n in ((0, x, y, N * T * H * W * G), (1, dy, dx, N * To * Ho * Wo * G)):
        scratch = torch.empty(n, dtype=F32T, device=DEV)
        _call('og_blurpool3d_grouped', src.data_ptr(), dst.ptr(), scratch.data_ptr(), bwd, N, T, H, W, cin, cout, G, k,
              st, sh, sw)
    torch.cuda.synchronize()
    y.check_guard('y')
    dx.check_guard('dx')
    _check('y', y.t, *grouped_expect(x, G, cout, k, stride, False))
    _check('dx', dx.t, *grouped_expect(dy, G, cin, k, stride, True, (T, H, W)))
    return x, dy, y.t, dx.t


GROUPED_CASES = [
    # (G, k, stride, (T, H, W), cin, cout)
    (1, 3, (1, 2, 2), (4, 9, 11), 64, 64),
    (2, 3, (1, 1, 1), (3, 7, 9), 64, 128),
    (2, 3, (2, 2, 2), (5, 9, 11), 128, 128),
    (4, 1, (2, 2, 2), (3, 5, 7), 64, 32),
    (4, 5, (1, 2, 2), (3, 3, 9), 128, 64),      # H < k
    (8, 3, (2, 4, 4), (5, 9, 13), 128, 128),    # stride > k: input voxels no tap reaches get exactly 0
    (8, 7, (2, 2, 2), (3, 7, 5), 64, 128),
    (8, 5, (1, 1, 1), (1, 5, 6), 64, 64),       # T = 1
    (16, 3, (2, 2, 2), (4, 8, 8), 128, 256),    # G = cin / 8
    (8, 3, (2, 4, 4), (6, 10, 17), 64, 64),     # G = cin / 8
    (2, 7, (1, 2, 2), (2, 6, 5), 48, 16),       # 24- and 8-channel groups
]


@GPU
@pytest.mark.parametrize('G,k,stride,thw,cin,cout', GROUPED_CASES)
def test_grouped_blurpool_against_float64(G, k, stride, thw, cin, cout):
    grouped_run(2, *thw, cin, cout, G, k, stride, 3100 + G + k + sum(thw))


@GPU
@pytest.mark.parametrize('k,stride,thw', [(3, (2, 2, 2), (4, 9, 11)), (5, (1, 2, 2), (3, 8, 8)), (1, (2, 4, 4), (3, 9, 7))])
def test_one_group_is_bit_identical_to_og_blurpool3d(k, stride, thw):
    x, dy, y, dx = grouped_run(2, *thw, 64, 128, 1, k, stride, 3200 + k)
    T, H, W = thw
    y1, dx1 = torch.empty_like(y), torch.empty_like(dx)
    To, Ho, Wo = y.shape[1:4]
    for bwd, src, dst, n in ((0, x, y1, 2 * T * H * W), (1, dy, dx1, 2 * To * Ho * Wo)):
        scratch = torch.empty(n, dtype=F32T, device=DEV)
        _call('og_blurpool3d', src.data_ptr(), dst.data_ptr(), scratch.data_ptr(), bwd, 2, T, H, W, 64, 128, k,
              *stride)
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), y1.view(torch.int16))
    assert torch.equal(dx.view(torch.int16), dx1.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------------
# module level
# ------------------------------------------------------------------------------------------------------------------
def _run(m, x):
    """Forward + backward of mean(y^2) through the CUDA path. Returns y (NCDHW fp32), dx and the parameter grads."""
    from open_genie_b200 import ops
    xg = x.clone().to(DEV).requires_grad_(True)
    y = m(xg)
    yr = ops.to_reference(y) if y.dim() == 5 else y
    g = (2.0 / y.numel()) * y.detach().float()
    y.backward(g.to(y.dtype))
    grads = {k: p.grad.float().cpu() for k, p in m.named_parameters() if p.grad is not None}
    return yr.float().cpu(), xg.grad.float().cpu(), grads


@GPU
@pytest.mark.parametrize('tag', BLOCKS + ('blur_g4', 'video_disc_g2'))
def test_case_against_golden_and_oracle(golden, tag):
    g = golden(GOLDEN)[tag]
    m, oracle = _case_module_and_oracle(tag, g)
    sd = det_weights(m)
    m.to(DEV)
    x = bf16_round(O.det_uniform(f'causal.x.{tag}', g['shape']))
    y, dx, grads = _run(m, x)
    assert tuple(y.shape) == g['y_shape']
    # against the oracle on what the kernels see: bf16 conv weights and input, fp32 math
    sdr = {k: v.clone().requires_grad_(True) for k, v in round_conv_weights(sd).items()}
    xo = x.clone().requires_grad_(True)
    yo = oracle(sdr, xo)
    yo.square().mean().backward()
    # the critic stacks a stem, two blocks scaled by 4 and a head, with bf16 activations between its kernels: its
    # gradients get the bounds test_gpu_gan.py gives the critic with one group
    deep = 3 if tag == 'video_disc_g2' else 1
    tol_y, tol_dx, tol_g = (3e-2, 0.12, 0.15) if tag == 'video_disc_g2' else (1e-2, 3e-2, 3e-2)
    assert rel_l2(y, yo.detach()) < tol_y, rel_l2(y, yo.detach())
    assert rel_l2(dx, xo.grad) < tol_dx, rel_l2(dx, xo.grad)
    assert set(grads) == set(g['grad_names'])
    for k in grads:
        if not _ill_conditioned(m, k):
            assert rel_l2(grads[k], sdr[k].grad) < tol_g, (k, rel_l2(grads[k], sdr[k].grad))
    # against the fp32 reference run on the unrounded input
    assert rel_l2(_sample(f'causal.y.{tag}', y, 256), g['y']) < 2e-2 * deep
    assert rel_l2(_sample(f'causal.dx.{tag}', dx, 256), g['dx']) < 5e-2 * deep
    for k, n in g['grad_norm'].items():
        if not _ill_conditioned(m, k):
            assert abs(grads[k].norm().item() - n) <= 5e-2 * deep * n + 1e-7, k


@GPU
@pytest.mark.parametrize('kw', [dict(in_channels=64, out_channels=128, use_causal=True),
                                dict(in_channels=128, num_groups=2, use_causal=True, act_fn='leaky'),
                                dict(in_channels=64, out_channels=128, kernel_size=1, use_causal=True)])
def test_fused_causal_block_matches_its_layers(kw):
    """The single fused node (no down-sampling, (C/G) % 8 == 0) against the same layers run one module at a time."""
    from open_genie_b200 import ops
    m = _block(kw)
    det_weights(m)
    m.to(DEV)
    x = bf16_round(O.det_uniform('causal.fused.x', (2, kw['in_channels'], 5, 8, 8))).to(DEV)
    xf = x.clone().requires_grad_(True)
    yf = m(xf)
    assert hasattr(yf, '_og_gn_sums')                  # only the fused node hands its output statistics on
    gup = O.det_uniform('causal.fused.g', tuple(yf.shape)).to(DEV)
    yf.backward(gup.to(yf.dtype))
    gf = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    xl = x.clone().requires_grad_(True)
    h = m.main[2](m.main[0](xl))
    yl = m.main[6].conv3d(m.main[4](h), x2=xl)
    yl.backward(gup.to(yl.dtype))
    assert rel_l2(ops.to_reference(yf).float(), ops.to_reference(yl).float()) < 5e-3
    assert rel_l2(xf.grad.float(), xl.grad.float()) < 2e-2
    for k, p in m.named_parameters():
        assert rel_l2(gf[k].float(), p.grad.float()) < 2e-2, k


@GPU
def test_fused_block_passes_the_time_padding_of_its_geometry():
    """og_conv3d_fwd receives pt = kt - 1 for a causal block and (kt - 1) // 2 for a plain one, in both convs."""
    from open_genie_b200 import _lib
    x = torch.randn((1, 64, 4, 8, 8), device=DEV)
    for causal, k, want in ((True, 3, 2), (False, 3, 1), (True, 5, 4), (False, 5, 2), (True, 1, 0)):
        m = _block(dict(in_channels=64, kernel_size=k, use_causal=causal)).to(DEV)
        _lib.TIMING = []
        try:
            m(x)
            calls = [c[1] for c in _lib.TIMING if c[0] == 'og_conv3d_fwd']
        finally:
            _lib.TIMING = None
        assert len(calls) == 2, calls
        for a in calls:
            assert a[2:8] == (k, k, k, want, (k - 1) // 2, (k - 1) // 2), (causal, k, a[2:8])


@GPU
def test_causal_block_runs_grouped_blur_and_plain_groups_keep_their_calls():
    """A down-sampling block with num_groups = 2 pools through og_blurpool3d_grouped; with num_groups = 1 it still
    calls og_blurpool3d with the arguments it always did."""
    from open_genie_b200 import _lib
    x = torch.randn((1, 64, 4, 8, 8), device=DEV, requires_grad=True)
    for G, use_causal in ((2, True), (1, False), (1, True)):
        m = _block(dict(in_channels=64, out_channels=128, downsample=2, num_groups=G, use_causal=use_causal)).to(DEV)
        _lib.TIMING = []
        try:
            m(x).float().sum().backward()
            torch.cuda.synchronize()
            calls = [(c[0], c[1]) for c in _lib.TIMING if 'blurpool' in c[0]]
        finally:
            _lib.TIMING = None
        assert len(calls) == 4, calls                # both branches, forward and backward
        if G == 1:
            assert all(n == 'og_blurpool3d' for n, _ in calls)
            assert sorted(a[8:14] for _, a in calls) == sorted([(64, 64, 3, 2, 2, 2), (128, 128, 3, 2, 2, 2)] * 2)
        else:
            assert all(n == 'og_blurpool3d_grouped' and a[10] == 2 for n, a in calls)


# ------------------------------------------------------------------------------------------------------------------
# model level: the causal mini tokenizer
# ------------------------------------------------------------------------------------------------------------------
def _tokenizer(t):
    import open_genie_b200 as og
    tok = og.VideoTokenizer(t['enc'], t['dec'], d_codebook=t['d_codebook'], gan_loss_weight=0, perc_loss_weight=0)
    sd = det_weights(tok)
    return tok.to(DEV), sd


@GPU
def test_causal_tokenizer_training_step_against_golden(golden):
    t = golden(GOLDEN)['tokenizer']
    tok, _ = _tokenizer(t)
    tok.train()
    video = O.det_uniform('causal.tokenizer.video', t['video_shape']).to(DEV)
    loss = tok.training_step(video, 0)
    loss.backward()
    _, (rec, _, _, _, ql) = tok(video)
    assert abs(rec.item() - t['rec_loss']) <= 2e-2 * t['rec_loss']
    assert abs(ql.item() - t['quant_loss']) <= 5e-2 * abs(t['quant_loss'])
    assert abs(loss.item() - t['loss']) <= 3e-2 * t['loss']
    grads = {k: p.grad.float().cpu() for k, p in tok.named_parameters() if p.grad is not None}
    assert set(grads) == set(t['grad_names'])
    # the decoder's gradients agree in norm and direction; the encoder's pass through the LFQ entropy at beta = 100,
    # narrower than bf16 noise on the latent (see test_gpu_tokenizer.py), so only their scale is compared
    for k, n in t['grad_norm'].items():
        if n <= 1e-6 or _ill_conditioned(tok, k):
            continue
        r = grads[k].norm().item() / n
        if k.startswith('dec_layers'):
            assert abs(r - 1) < 5e-2, (k, r)
            assert rel_l2(_sample(f'causal.tok.g.{k}', grads[k], 32), t['grad'][k]) < 0.1, k
        else:
            assert 0.5 < r < 2.0, (k, r)


@GPU
def test_causal_tokenizer_tokenize_decode_and_encoder_chain(golden):
    from open_genie_b200 import ops
    t = golden(GOLDEN)['tokenizer']
    tok, sd = _tokenizer(t)
    video = O.det_uniform('causal.tokenizer.video', t['video_shape']).to(DEV)
    quant, idxs = tok.tokenize(video)
    assert tuple(quant.shape) == t['quant_shape'] and idxs.shape == t['idxs'].shape and idxs.dtype == torch.int64
    safe = (t['enc_latent'].abs() > 0.05 * t['enc_latent'].abs().mean()).all(1)
    assert (idxs.cpu()[safe] == t['idxs'][safe]).float().mean().item() > 0.97
    dec = tok.decode(quant)
    assert tuple(dec.shape) == t['decode_shape'] and dec.dtype == torch.float32
    # the encoder against the oracle on bf16-rounded weights and input
    vb = bf16_round(video.cpu())
    enc = ops.to_reference(tok.encode(vb.to(DEV))).float().cpu()
    enc_o = C.run_layers(round_conv_weights(sd), 'enc_layers', t['enc'], vb)
    assert enc.shape == enc_o.shape == t['enc_shape']
    assert rel_l2(enc, enc_o) < 2e-2, rel_l2(enc, enc_o)


@GPU
def test_causal_tokenizer_graphed_step_matches_eager(golden):
    from open_genie_b200 import ops
    from open_genie_b200.graph import GraphedTrainStep
    t = golden(GOLDEN)['tokenizer']
    video = O.det_uniform('causal.tokenizer.video', t['video_shape']).to(DEV)
    try:
        tok, _ = _tokenizer(t)
        step = GraphedTrainStep(tok, tok.configure_optimizers(), video, warmup=2)
        with torch.no_grad():
            expect = float(tok.training_step(video, 0))
        got = step(video).item()
        assert abs(got - expect) <= 5e-3 * abs(expect), (got, expect)
        with torch.no_grad():
            after = float(tok.training_step(video, 0))
        assert after != got
    finally:
        ops.enable_zero_arena(False)
