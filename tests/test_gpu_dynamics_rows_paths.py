"""The row kernels of DynamicsModel (csrc/dynamics_rows.cu) against explicit float64 references, element by element.

Paths covered: og_embed_add_fwd / og_embed_add_bwd (C = 8 and 512, T > 1 so that rows_per_act = H W, every token
the same id, vocabularies of 1, enough rows for the grid-stride loops); og_masked_ce_fwd / og_masked_ce_bwd (V from 1
to 16384, V not a multiple of 32, all / no / one / alternating rows masked, the target at the row maximum and far
below it, logits of magnitude 1e3, gloss != 1, 32768 rows) and the autograd function of ops.py; og_softmax_cdf (bf16
and fp32 logits, inv_temp 0.5 / 1 / 2, V = 1, 31, 33, 1024, logits of standard deviation 1, 4 and 16); and
og_maskgit_sample against a Python mirror of its rule fed the kernel's own CDF (bit exact on codes and mask), and
against the reference's semantics, confidence = prob[pred] in float64 (P not a power of two, P = 4096, B > 1,
confidence ties, k larger than the positions still masked, more steps than needed, peaked logits).

Every tolerance is a worst-case bound built from the rounding points of the kernel under test. The
`test_tolerance_rejects_*` tests run on the CPU and show that each bound still rejects the mistakes it exists to catch.
Out-of-range token, action and target indices make the kernels trap; those paths are not launched here.
"""
import ctypes

import pytest
import torch

GPU = pytest.mark.gpu
DEV = 'cuda'
F32T, F64T, BF16 = torch.float32, torch.float64, torch.bfloat16

# Rounding model, as in test_gpu_attention_paths.py: U is the bf16 unit roundoff, F32 one fp32 ulp per operation, and
# a sequential fp32 sum of n terms is within gam(n) of the exact sum relative to the sum of the terms' magnitudes.
U = 2.0 ** -8
F32 = 2.0 ** -23
SLACK = 1.02
TINY = 2.0 ** -100
# CUDA C Programming Guide, intrinsic functions: __expf(x) is within 2 + floor(|1.173 x|) ulp; __logf(x) has an absolute
# error of at most 2^-21.41 for x in [0.5, 2] and 3 ulp elsewhere. expf (used by og_softmax_cdf) is within 2 ulp.
LOGF_ABS = 2.0 ** -21.41


def gam(n):
    return n * F32



def check(name, got, ref, tol):
    got = got.double().to(ref.device)
    assert got.shape == ref.shape, f'{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
    tol = tol + TINY
    bad = ~(err <= tol)    # NaN (an element never written) is bad too
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        ratio = (err / tol).flatten().nan_to_num(float('inf')).max().item()
        raise AssertionError(
            f'{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound, worst err/tol {ratio:.3g}; first at '
            f'flat index {i} (of shape {tuple(ref.shape)}): got {got.flatten()[i].item():.8g}, '
            f'ref {ref.flatten()[i].item():.8g}, tol {tol.flatten()[i].item():.3g}')


def _rejects(name, got, ref, tol):
    with pytest.raises(AssertionError):
        check(name, got, ref, tol)


# ------------------------------------------------------------------------------------------------------------------
# float64 references and bounds
# ------------------------------------------------------------------------------------------------------------------
def embed_bwd_expect(tok, act, dy, tok_vocab, act_vocab, rows_per_act):
    """index_add of dy (bf16 [rows, C], exact in float64) into zeroed fp32 tables. Each table row is an fp32 sum, by
    atomics in any order, of `count` values: within gam(count) of the exact sum, relative to the sum of |dy|."""
    dy = dy.double()
    a_rows = act.repeat_interleave(rows_per_act)
    out = {}
    for name, idx, vocab in (('d_tok_w', tok, tok_vocab), ('d_act_w', a_rows, act_vocab)):
        ref = torch.zeros(vocab, dy.shape[1], dtype=F64T, device=dy.device).index_add_(0, idx, dy)
        mag = torch.zeros_like(ref).index_add_(0, idx, dy.abs())
        cnt = torch.bincount(idx, minlength=vocab).to(F64T)[:, None]
        out[name] = (ref, SLACK * gam(cnt) * mag)
    return out


def masked_ce_expect(logits, target, mask, gloss=1.0, mut=()):
    """float64 log-softmax of the bf16 logits. Returns loss, dlogits (each (ref, tol)).
    Bounds: lse = m + __logf(s), s = sum_j __expf(l_j - m) in 32 lanes of V/32 terms and a 5-level tree; each exp term is
    off by (2 + 1.173 |l_j - m|) F32 relatively, s by gam(V/32 + 5) more, s lies in [1, V] so __logf adds 2^-21.41
    (s <= 2) or 3 ulp of log s, and m + log s one rounding. loss = sum (lse - l_t) / count: the per-row terms are
    summed per warp then with atomics in any order, and the final division rounds once.
    dlogits = bf16(g (__expf(l - lse) - [j = t])), g = gloss / count: the exponent is off by the lse error plus the
    subtraction's rounding, __expf by (2 + 1.173 |l - lse|) ulp, then two products and the bf16 rounding.
    `mut` 'no_onehot' drops the target term's one-hot (only the sensitivity test passes it)."""
    l = logits.double()
    rows, V = l.shape
    sel = mask.bool()
    m = l.amax(1, keepdim=True)
    x = l - m
    s = x.exp().sum(1, keepdim=True)
    lse = m + s.log()
    e_s = ((x.exp() * (2 + 1.173 * x.abs())).sum(1, keepdim=True) * F32 + gam(V // 32 + 6) * s) / s
    ls = s.log()
    e_log = torch.where(s <= 2, torch.full_like(s, LOGF_ABS), 3 * F32 * ls.abs())
    e_lse = e_s + e_log + F32 * lse.abs()
    lt = l.gather(1, target[:, None])
    term = (lse - lt).squeeze(1)[sel]
    count = int(sel.sum())
    loss = term.sum() / count if count else torch.tensor(float('nan'), dtype=F64T)
    e_loss = ((e_lse + F32 * (lse - lt).abs()).squeeze(1)[sel].sum() + gam(rows) * term.abs().sum()) / max(count, 1) \
        + F32 * abs(float(loss) if count else 0.0)
    g = gloss / max(count, 1)
    p = (l - lse).exp()
    onehot = torch.zeros_like(l).scatter_(1, target[:, None], 1.0)
    if 'no_onehot' in mut:
        onehot.zero_()
    d = g * (p - onehot)
    d = torch.where(sel[:, None], d, torch.zeros_like(d))
    e_p = p * (e_lse + F32 * (l - lse).abs() + (2 + 1.173 * (l - lse).abs()) * F32)
    e_d = abs(g) * (e_p + gam(3) * (p + onehot)) + U * d.abs()
    e_d = torch.where(sel[:, None], e_d, torch.zeros_like(e_d))
    return {'loss': (loss, SLACK * e_loss), 'dlogits': (d, SLACK * e_d)}


def cdf_expect(logits, inv_temp, mut=()):
    """float64 cumulative softmax of the exact scaled logits (inv_temp is a power of two: the scaling is exact).
    Each p_j = expf(x_j - m) / s: the subtraction rounds (|x_j - m| F32 / 2 relatively after exp), expf 2 ulp, s is a
    32-lane sum of V/32 terms plus a 5-level tree (gam(V/32 + 5)), 1/s and the product one rounding each. The scan
    adds at most 5 tree levels and one carry per 32-entry chunk: gam(V/32 + 6) of the running sum. The running
    maximum keeps each entry within the largest bound before it, and the bound is non-decreasing.
    `mut` 'exclusive' shifts the reference by one entry (an exclusive scan)."""
    x = logits.double() * inv_temp
    V = x.shape[1]
    m = x.amax(1, keepdim=True)
    p = (x - m).exp()
    p = p / p.sum(1, keepdim=True)
    rho = gam(V // 32 + 10) + F32 * (x - m).abs()
    ref = p.cumsum(1)
    if 'exclusive' in mut:
        ref = ref - p
    tol = (p * rho).cumsum(1) + gam(V // 32 + 6) * ref.abs()
    return ref, SLACK * tol, p, rho


def _cpu(shape, seed, std=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * std


# ------------------------------------------------------------------------------------------------------------------
# CPU: each bound rejects the mistakes it exists for
# ------------------------------------------------------------------------------------------------------------------
def test_tolerance_rejects_masked_ce_mistakes():
    rows, V = 40, 33
    lg = _cpu((rows, V), 1, 3.0).to(BF16)
    tgt = torch.randint(0, V, (rows,), generator=torch.Generator().manual_seed(2))
    mask = torch.arange(rows) % 2 == 0
    ex = masked_ce_expect(lg, tgt, mask, 0.7)
    check('loss', ex['loss'][0].float(), *ex['loss'])
    check('dlogits', ex['dlogits'][0].to(BF16), *ex['dlogits'])
    # loss over every row instead of the masked ones; mean over all rows; the log-sum-exp without its maximum shift
    _rejects('loss', masked_ce_expect(lg, tgt, torch.ones(rows, dtype=torch.bool), 0.7)['loss'][0].float(), *ex['loss'])
    _rejects('loss', (ex['loss'][0] * int(mask.sum()) / rows).float(), *ex['loss'])
    _rejects('dlogits', masked_ce_expect(lg, tgt, mask, 0.7, mut=('no_onehot',))['dlogits'][0].to(BF16),
             *ex['dlogits'])
    # gloss ignored
    _rejects('dlogits', masked_ce_expect(lg, tgt, mask, 1.0)['dlogits'][0].to(BF16), *ex['dlogits'])


def test_tolerance_rejects_cdf_mistakes():
    lg = _cpu((8, 1024), 3, 4.0)
    ref, tol, p, _ = cdf_expect(lg, 1.0)
    check('cdf', ref.float(), ref, tol)
    _rejects('cdf', cdf_expect(lg, 1.0, mut=('exclusive',))[0].float(), ref, tol)
    _rejects('cdf', cdf_expect(lg, 0.5)[0].float(), ref, tol)               # temperature applied the wrong way
    # a whole 32-entry chunk's carry dropped
    bad = ref.clone()
    bad[:, 64:] -= ref[:, 31:32]
    _rejects('cdf', bad.float(), ref, tol)


def test_tolerance_rejects_embedding_gradient_mistakes():
    rows, C = 64, 16
    tok = torch.randint(0, 5, (rows,), generator=torch.Generator().manual_seed(4))
    act = torch.randint(0, 3, (rows // 8,), generator=torch.Generator().manual_seed(5))
    dy = _cpu((rows, C), 6).to(BF16)
    ex = embed_bwd_expect(tok, act, dy, 5, 3, 8)
    check('d_tok_w', ex['d_tok_w'][0].float(), *ex['d_tok_w'])
    # each frame's rows given the next frame's action
    bad = embed_bwd_expect(tok, act.roll(1), dy, 5, 3, 8)
    _rejects('d_act_w', bad['d_act_w'][0].float(), *ex['d_act_w'])
    # one row dropped (a grid-stride loop that stops one step early)
    short = dy.clone()
    short[-1] = 0
    bad = embed_bwd_expect(tok, act, short, 5, 3, 8)
    _rejects('d_tok_w', bad['d_tok_w'][0].float(), *ex['d_tok_w'])


# ------------------------------------------------------------------------------------------------------------------
# CPU: host-side argument validation
# ------------------------------------------------------------------------------------------------------------------
def test_dynamics_rows_argument_validation_returns_status_codes():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error())
    bad(lib.og_embed_add_fwd(p, p, p, p, p, 4, 2, 12, 8, 8, None), b'multiple of 8')
    bad(lib.og_embed_add_bwd(p, p, p, p, p, 4, 2, 12, 8, 8, None), b'multiple of 8')
    bad(lib.og_embed_add_fwd(p, p, p, p, p, 0, 2, 16, 8, 8, None), b'bad arguments')
    bad(lib.og_embed_add_fwd(p, p, p, p, p, 4, 0, 16, 8, 8, None), b'bad arguments')
    bad(lib.og_masked_ce_fwd(p, p, p, 4, 0, p, p, None), b'bad arguments')
    bad(lib.og_masked_ce_bwd(p, p, p, p, p, None, None, 4, 8, None), b'bad arguments')
    bad(lib.og_softmax_cdf(p, 0, 4, 0, 1.0, p, p, None), b'bad arguments')
    for P in (0, 4097):
        bad(lib.og_maskgit_sample(p, p, 0, 1.0, p, p, p, 1, 1, P, 8, p, p, None), b'positions per frame')
    bad(lib.og_maskgit_sample(p, p, 0, 1.0, None, p, p, 1, 1, 16, 8, p, p, None), b'bad arguments')
    bad(lib.og_maskgit_sample(p, p, 0, 1.0, p, p, p, 0, 1, 16, 8, p, p, None), b'bad arguments')


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------
# GPU: embedding sum
# ------------------------------------------------------------------------------------------------------------------
EMBED = {  # name: (B, T, H, W, C, tok_vocab, act_vocab, same_id)
    'c8': (2, 3, 4, 4, 8, 17, 5, False),
    'c512_t4': (2, 4, 8, 8, 512, 1024, 8, False),
    'hot_row': (2, 4, 16, 16, 512, 1024, 8, True),
    'vocab_1': (1, 2, 4, 4, 64, 1, 1, False),
    'grid_stride': (8, 16, 16, 16, 512, 1024, 8, False),     # 32768 rows x 64 vectors: > 132 * 16 * 256 threads
}


@GPU
@pytest.mark.parametrize('case', list(EMBED))
def test_embed_add(case):
    B, T, H, W, C, tv, av, same = EMBED[case]
    rows = B * T * H * W
    g = _gen(100 + len(case))
    tok = torch.randint(0, tv, (rows,), generator=g, device=DEV)
    if same:
        tok.fill_(tv // 3)
    act = torch.randint(0, av, (B * T,), generator=g, device=DEV)
    tok_w = torch.randn((tv, C), generator=g, device=DEV)
    act_w = torch.randn((av, C), generator=g, device=DEV)
    out = torch.full((rows + 1, C), float('nan'), dtype=BF16, device=DEV)      # one guard row
    _call('og_embed_add_fwd', tok.data_ptr(), act.data_ptr(), tok_w.data_ptr(), act_w.data_ptr(), out.data_ptr(), rows,
          H * W, C, tv, av)
    ref = (tok_w[tok] + act_w[act.repeat_interleave(H * W)]).to(BF16)         # bf16(fp32 sum): one rounding each
    assert torch.equal(out[:rows], ref)
    assert bool(out[rows].isnan().all())
    dy = torch.randn((rows, C), generator=g, device=DEV).to(BF16)
    dt = torch.zeros((tv, C), dtype=F32T, device=DEV)
    da = torch.zeros((av, C), dtype=F32T, device=DEV)
    _call('og_embed_add_bwd', tok.data_ptr(), act.data_ptr(), dy.data_ptr(), dt.data_ptr(), da.data_ptr(), rows, H * W,
          C, tv, av)
    ex = embed_bwd_expect(tok, act, dy, tv, av, H * W)
    check('d_tok_w', dt, *ex['d_tok_w'])
    check('d_act_w', da, *ex['d_act_w'])


# ------------------------------------------------------------------------------------------------------------------
# GPU: masked cross entropy
# ------------------------------------------------------------------------------------------------------------------
def _ce_inputs(rows, V, mask_kind, seed, scale=3.0, target_kind='random'):
    g = _gen(seed)
    lg = (torch.randn((rows, V), generator=g, device=DEV) * scale).to(BF16)
    if target_kind == 'max':
        tgt = lg.float().argmax(1)
    elif target_kind == 'far':
        tgt = torch.randint(0, V, (rows,), generator=g, device=DEV)
        lg[torch.arange(rows, device=DEV), tgt] = -30.0 * scale            # far below the row maximum
    else:
        tgt = torch.randint(0, V, (rows,), generator=g, device=DEV)
    r = torch.arange(rows, device=DEV)
    mask = {'all': torch.ones(rows, dtype=torch.bool, device=DEV),
            'none': torch.zeros(rows, dtype=torch.bool, device=DEV),
            'one': r == rows // 2,
            'alternate': r % 2 == 1,
            'random': torch.rand(rows, generator=g, device=DEV) < 0.4}[mask_kind]
    return lg, tgt, mask


def ce_run(lg, tgt, mask, gloss):
    rows, V = lg.shape
    m8 = mask.to(torch.uint8)
    row_lse = torch.full((rows,), float('nan'), dtype=F32T, device=DEV)
    stats = torch.zeros(2, dtype=F32T, device=DEV)
    _call('og_masked_ce_fwd', lg.data_ptr(), tgt.data_ptr(), m8.data_ptr(), rows, V, row_lse.data_ptr(),
          stats.data_ptr())
    gl = torch.tensor([gloss], dtype=F32T, device=DEV)
    dl = torch.full((rows, V), float('nan'), dtype=BF16, device=DEV)
    _call('og_masked_ce_bwd', lg.data_ptr(), tgt.data_ptr(), m8.data_ptr(), row_lse.data_ptr(), stats.data_ptr(),
          gl.data_ptr(), dl.data_ptr(), rows, V)
    torch.cuda.synchronize()
    return stats, dl


CE = [  # rows, V, mask, scale, target
    (64, 1, 'all', 3.0, 'random'), (64, 33, 'alternate', 3.0, 'random'), (100, 1000, 'random', 3.0, 'far'),
    (100, 1024, 'one', 3.0, 'max'), (64, 16384, 'alternate', 3.0, 'random'), (64, 1024, 'none', 3.0, 'random'),
    (64, 1024, 'all', 1e3, 'random'), (64, 1024, 'all', 1e3, 'far'), (64, 31, 'all', 3.0, 'max'),
    (32768, 1024, 'random', 3.0, 'random'),
]


@GPU
@pytest.mark.parametrize('rows,V,mask_kind,scale,target_kind', CE)
def test_masked_ce(rows, V, mask_kind, scale, target_kind):
    lg, tgt, mask = _ce_inputs(rows, V, mask_kind, 200 + V + rows, scale, target_kind)
    gloss = 0.37
    stats, dl = ce_run(lg, tgt, mask, gloss)
    count = int(mask.sum())
    assert stats[1].item() == count
    ex = masked_ce_expect(lg, tgt, mask, gloss)
    if count:
        check('loss', stats[0] / stats[1], *ex['loss'])
    check('dlogits', dl, *ex['dlogits'])
    assert bool((dl[~mask] == 0).all())                   # exactly zero (not NaN) on rows outside the mask


@GPU
def test_masked_ce_autograd_with_no_row_masked():
    """cross_entropy(logits[mask], ...) over an empty selection is NaN with zero gradients; so is the wrapper."""
    from open_genie_b200 import ops
    lg, tgt, mask = _ce_inputs(48, 100, 'none', 300)
    x = lg.clone().requires_grad_(True)
    loss = ops.masked_cross_entropy(x, tgt, mask)
    loss.backward()
    assert bool(torch.isnan(loss)) and bool((x.grad == 0).all())
    lr = lg.float().clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lr[mask], tgt[mask])
    ref.backward()
    assert bool(torch.isnan(ref)) and bool((lr.grad == 0).all())
    # and with rows masked, the same function as the C ABI
    lg, tgt, mask = _ce_inputs(48, 100, 'alternate', 301)
    x = lg.clone().requires_grad_(True)
    loss = ops.masked_cross_entropy(x, tgt, mask)
    (loss * 2.5).backward()
    ex = masked_ce_expect(lg, tgt, mask, 2.5)
    check('loss', loss, *ex['loss'])
    check('dlogits', x.grad, *ex['dlogits'])


# ------------------------------------------------------------------------------------------------------------------
# GPU: softmax CDF
# ------------------------------------------------------------------------------------------------------------------
def cdf_run(lg, inv_temp):
    rows, V = lg.shape
    cdf = torch.full((rows, V), float('nan'), dtype=F32T, device=DEV)
    st = torch.full((rows, 2), float('nan'), dtype=F32T, device=DEV)
    _call('og_softmax_cdf', lg.data_ptr(), int(lg.dtype == F32T), rows, V, inv_temp, cdf.data_ptr(), st.data_ptr())
    torch.cuda.synchronize()
    return cdf, st


@GPU
@pytest.mark.parametrize('dtype', [BF16, F32T])
@pytest.mark.parametrize('inv_temp', [0.5, 1.0, 2.0])
@pytest.mark.parametrize('V', [1, 31, 33, 1024])
@pytest.mark.parametrize('std', [1.0, 4.0, 16.0])
def test_softmax_cdf(dtype, inv_temp, V, std):
    rows = 200
    lg = (torch.randn((rows, V), generator=_gen(400 + V), device=DEV) * std).to(dtype)
    cdf, st = cdf_run(lg, inv_temp)
    ref, tol, p, _ = cdf_expect(lg, inv_temp)
    check('cdf', cdf, ref, tol)
    check('cdf[-1]', cdf[:, -1], torch.ones_like(ref[:, -1]), tol[:, -1])
    steps = cdf[:, 1:] - cdf[:, :-1]
    assert bool((steps >= 0).all()), f'{int((steps < 0).any(1).sum())}/{rows} rows step backwards'
    # row statistics: the exact maximum of the scaled logits and 1 / sum within the sum's bound
    x = lg.double() * inv_temp
    assert torch.equal(st[:, 0].double(), x.amax(1))
    e = (x - x.amax(1, keepdim=True)).exp()
    s = e.sum(1)
    # each term off by (2 + |x - m| / 2) ulp of itself (expf, the rounded argument), the sum by gam(V/32 + 5), 1/s once
    rel = (e * (2 + (x - x.amax(1, keepdim=True)).abs())).sum(1) * F32 / s + gam(V // 32 + 6)
    check('1/sum', st[:, 1], 1 / s, SLACK * rel / s)


# ------------------------------------------------------------------------------------------------------------------
# GPU: MaskGIT sampler
# ------------------------------------------------------------------------------------------------------------------
def sample_run(lg, uniforms, schedule, inv_temp=1.0):
    """og_softmax_cdf + og_maskgit_sample on logits [B, P, V]; returns code, mask, cdf, row_stats."""
    B, P, V = lg.shape
    cdf = torch.empty((B * P, V), dtype=F32T, device=DEV)
    st = torch.empty((B * P, 2), dtype=F32T, device=DEV)
    f32 = int(lg.dtype == F32T)
    _call('og_softmax_cdf', lg.data_ptr(), f32, B * P, V, inv_temp, cdf.data_ptr(), st.data_ptr())
    code = torch.full((B, P), -1, dtype=torch.int64, device=DEV)
    mask = torch.ones((B, P), dtype=torch.uint8, device=DEV)
    sch = torch.tensor(schedule, dtype=torch.int32, device=DEV)
    _call('og_maskgit_sample', cdf.data_ptr(), lg.data_ptr(), f32, inv_temp, st.data_ptr(), uniforms.data_ptr(),
          sch.data_ptr(), len(schedule), B, P, V, code.data_ptr(), mask.data_ptr())
    torch.cuda.synchronize()
    return code, mask, cdf.view(B, P, V), st.view(B, P, 2)


def maskgit_mirror(lg, cdf, st, uniforms, schedule, inv_temp=1.0):
    """The sampler's documented rule in Python, on the kernel's own CDF and row statistics:
    per row, while anything is masked: pred = first j with cdf[j] > u * cdf[V-1]; confidence = expf(logit[pred] *
    inv_temp - max) * (1/sum), -inf where already predicted; the k = schedule[s] first positions by (confidence
    descending, position ascending) get code = pred and mask = 0. Also returns, per step, the predictions and the
    masks before the step (for the reference-semantics check)."""
    B, P, V = cdf.shape
    code = torch.full((B, P), -1, dtype=torch.int64, device=DEV)
    mask = torch.ones((B, P), dtype=torch.bool, device=DEV)
    pos = torch.arange(P, device=DEV)
    trace = []
    for s, k in enumerate(schedule):
        for b in range(B):
            if not bool(mask[b].any()):
                continue
            u = uniforms[s, b] * cdf[b, :, V - 1]
            pred = torch.searchsorted(cdf[b], u[:, None].contiguous(), right=True).squeeze(1).clamp(max=V - 1)
            x = lg[b].float().gather(1, pred[:, None]).squeeze(1) * inv_temp
            conf = torch.exp(x - st[b, :, 0]) * st[b, :, 1]
            conf = torch.where(mask[b], conf, torch.full_like(conf, float('-inf'))).tolist()
            order = sorted(range(P), key=lambda i: (-conf[i], i))
            pick = torch.tensor(order[:min(k, P)], dtype=torch.long, device=DEV)
            trace.append((s, b, pred.clone(), mask[b].clone(), pick))
            code[b, pick] = pred[pick]
            mask[b, pick] = False
    return code, mask, trace


def check_reference_semantics(lg, trace, inv_temp=1.0):
    """At every step, the positions the kernel fixed are a top-k of prob[pred] computed in float64 (reference
    dynamics.py:146-152), up to the fp32 confidence's own error: conf_a (1 + rho_a) >= conf_b (1 - rho_b) for every
    picked a and every still-masked b that was not picked."""
    B, P, V = lg.shape
    x = lg.double() * inv_temp
    m = x.amax(2, keepdim=True)
    prob = (x - m).exp()
    prob = prob / prob.sum(2, keepdim=True)
    rho = gam(V // 32 + 10) + F32 * (x - m).abs()
    for s, b, pred, masked, pick in trace:
        c = prob[b].gather(1, pred[:, None]).squeeze(1)
        r = rho[b].gather(1, pred[:, None]).squeeze(1)
        picked = torch.zeros(P, dtype=torch.bool, device=DEV)
        picked[pick] = True
        a = picked & masked
        rest = masked & ~picked
        if not bool(a.any()) or not bool(rest.any()):
            continue
        lo = (c[a] * (1 + r[a])).min()
        hi = (c[rest] * (1 - r[rest])).max()
        assert bool(lo >= hi), (f'step {s} row {b}: a picked position has prob[pred] {float(c[a].min()):.9g}, an '
                                f'unpicked masked one {float(c[rest].max()):.9g}')


def _schedule(P, steps):
    base = [P // steps] * steps
    base[-1] += P - sum(base)
    return base


SAMPLE = {  # name: (B, P, V, std, schedule)
    'p100_b3': (3, 100, 64, 1.0, _schedule(100, 7)),
    'p4096': (1, 4096, 64, 2.0, _schedule(4096, 12)),
    'peaked4': (2, 256, 1024, 4.0, _schedule(256, 25)),
    'peaked16': (2, 256, 1024, 16.0, _schedule(256, 10)),
    'k_exceeds_masked': (2, 96, 33, 1.0, [90, 20, 50]),          # step 2 asks for 20 of 6 left
    'early_stop': (2, 64, 31, 1.0, [40, 24, 10, 10, 10]),       # nothing left after step 2
}


@GPU
@pytest.mark.parametrize('case', list(SAMPLE))
def test_maskgit_sample(case):
    B, P, V, std, schedule = SAMPLE[case]
    g = _gen(500 + P + V)
    lg = (torch.randn((B, P, V), generator=g, device=DEV) * std).to(BF16)
    uni = torch.rand((len(schedule), B, P), generator=g, device=DEV)
    code, mask, cdf, st = sample_run(lg, uni, schedule)
    mcode, mmask, trace = maskgit_mirror(lg, cdf, st, uni, schedule)
    assert torch.equal(code, mcode)
    assert torch.equal(mask.bool(), mmask)
    if sum(schedule) >= P:
        assert int(mask.sum()) == 0 and int(code.min()) >= 0
    check_reference_semantics(lg, trace)


@GPU
def test_maskgit_sample_confidence_ties():
    """Identical logits at every position and identical uniforms: every confidence ties, so the positions are fixed
    in ascending order, k per step."""
    B, P, V = 2, 50, 40
    row = torch.randn(V, generator=_gen(600), device=DEV)
    lg = row.expand(B, P, V).contiguous()
    uni = torch.full((4, B, P), 0.3, device=DEV)
    schedule = [13, 13, 13, 11]
    code, mask, cdf, st = sample_run(lg, uni, schedule)
    mcode, mmask, trace = maskgit_mirror(lg, cdf, st, uni, schedule)
    assert torch.equal(code, mcode) and torch.equal(mask.bool(), mmask)
    for s, b, pred, masked, pick in trace:
        start = sum(schedule[:s])
        assert pick.tolist() == list(range(start, min(start + schedule[s], P)))


@GPU
def test_maskgit_confidence_of_unlikely_draws():
    """Each position draws its last token (u close to 1), whose probability is ~1e-5 and differs between positions
    by 1e-4 relatively. A confidence taken as cdf[j] - cdf[j-1] near cdf = 1 is quantised to 2^-24 ~ 6e-8, i.e. 0.6 %
    of these values, and would fix the positions in a scrambled order; prob[pred] keeps the order."""
    B, P, V = 2, 512, 64
    g = torch.Generator().manual_seed(700)
    rank = torch.stack([torch.randperm(P, generator=g) for _ in range(B)]).double()
    p_last = 1e-5 * (1 + 1e-4 * rank)
    lg = torch.zeros((B, P, V), dtype=F64T)
    lg[:, :, V - 1] = torch.log(p_last * (V - 1) / (1 - p_last))
    lg = lg.float().to(DEV)
    uni = torch.full((4, B, P), 1 - 2.0 ** -20, device=DEV)
    schedule = [P // 4] * 4
    code, mask, cdf, st = sample_run(lg, uni, schedule)
    assert bool((code == V - 1).all())
    mcode, mmask, trace = maskgit_mirror(lg, cdf, st, uni, schedule)
    assert torch.equal(code, mcode) and torch.equal(mask.bool(), mmask)
    check_reference_semantics(lg, trace)
    # positions are fixed from the most to the least likely draw
    for s, b, pred, masked, pick in trace:
        assert set(pick.tolist()) == set(torch.argsort(-rank[b])[s * P // 4:(s + 1) * P // 4].tolist())


@GPU
def test_ops_maskgit_sample_matches_c_abi():
    from open_genie_b200 import ops
    B, h, w, V = 2, 8, 12, 1024
    g = _gen(800)
    lg = (torch.randn((B, h, w, V), generator=g, device=DEV) * 4).to(BF16)
    uni = torch.rand((6, B * h * w), generator=g, device=DEV)
    sch = torch.tensor(_schedule(h * w, 6))
    code, mask = ops.maskgit_sample(lg, uni, sch)
    c2, m2, _, _ = sample_run(lg.view(B, h * w, V), uni.view(6, B, h * w), sch.tolist())
    assert torch.equal(code.view(B, -1), c2) and int(mask.sum()) == 0


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
@GPU
def test_dispatch_kernel_names():
    """The cases above reach every kernel of dynamics_rows.cu (only the launches run under the profiler)."""
    from test_gpu_attention_paths import _kernels_run
    g = _gen(900)
    rows, C, V = 64, 8, 33
    tok = torch.randint(0, 17, (rows,), generator=g, device=DEV)
    act = torch.randint(0, 5, (rows // 16,), generator=g, device=DEV)
    tok_w, act_w = torch.randn((17, C), device=DEV), torch.randn((5, C), device=DEV)
    out = torch.empty((rows, C), dtype=BF16, device=DEV)
    dt, da = torch.zeros((17, C), device=DEV), torch.zeros((5, C), device=DEV)
    lg, tgt, mask = _ce_inputs(rows, V, 'alternate', 901)
    lb = lg.view(1, rows, V)
    uni = torch.rand((2, 1, rows), generator=g, device=DEV)
    torch.cuda.synchronize()

    def run():
        _call('og_embed_add_fwd', tok.data_ptr(), act.data_ptr(), tok_w.data_ptr(), act_w.data_ptr(), out.data_ptr(),
              rows, 16, C, 17, 5)
        _call('og_embed_add_bwd', tok.data_ptr(), act.data_ptr(), out.data_ptr(), dt.data_ptr(), da.data_ptr(), rows, 16,
              C, 17, 5)
        ce_run(lg, tgt, mask, 1.0)
        sample_run(lb, uni, [rows // 2, rows // 2])
    names = _kernels_run(run)
    for w in ('og_embed_add_fwd_kernel', 'og_embed_add_bwd_kernel', 'og_masked_ce_fwd_kernel',
              'og_masked_ce_bwd_kernel', 'og_softmax_cdf_kernel', 'og_maskgit_sample_kernel'):
        assert any(w in n for n in names), (w, sorted(set(n for n in names if 'og_' in n)))
