"""Every path of the convolution weight gradient (og_conv3d_wgrad, og_conv3d_wgrad_bias, og_conv3d_strided_wgrad) and of
the strided forward and data gradient (og_conv3d_strided_fwd, og_conv3d_strided_dgrad) through the C ABI, against one
float64 "convolution by taps" reference.

Two kinds of check:
- Exact. x, dy and w are small integers and every output element's sum of |terms| (initial value included) stays below
  2^22, so every partial sum, in any order and any split, is an integer fp32 holds exactly. The kernels' dW, db and fp32
  outputs must then EQUAL the float64 reference, and bf16 outputs must equal its rounding to bf16. A dropped, doubled
  or shifted 64-voxel k-step, a stream-K segment added twice, a wrong tap, panel or row all change an integer. This
  assumes wgmma's fp32 accumulation keeps every bit of integer partial sums below 2^24.
- Bounded. Real operands with exponents spread over 2^+-10 and random signs, and per-element bounds
  gam(n) * sum|terms| with n = reduction length + stream-K segments + 1 (the += into the initial value, whose
  magnitude is included), plus U * |ref| for bf16 outputs. These catch type and descriptor errors that integer data
  cannot (bf16 read as fp16, a wrong swizzle on one panel).

Every output sits in a NaN-filled `Guarded` buffer (the weight-gradient workspace too, so an unwritten slot or bias
partial shows), accumulated outputs start from non-zero values, and every case runs twice and must give the same bits.

A Python mirror of launch_wgrad's host arithmetic (`WgradPlan`) says which schedule path each weight-gradient case
takes on the running device (its SM count), and each case checks the mirror's launch count against the library's.
CPU tests check the reference against torch, the mirror's invariants at several SM counts, that the bounds and the
integer data reject the mistakes they exist for, and that every argument check returns -1 before any CUDA call.
"""
import ctypes
import itertools
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from conv_ref import (BF16, DEV, EXACT_LIMIT, F32T, F64T, SLACK, U, cdiv, check, check_exact, dgrad_ref, fwd_ref, gam,
                      operand, torch_ref, voxel_box, wgrad_ref)
from conv_ref import nan_bits as _nan_bits
from conv_ref import rejects as _rejects
from helpers import Guarded

GPU = pytest.mark.gpu

SCRATCH = 64 << 20          # the step scope's reduction scratch (ops.StepScope.SCRATCH_BYTES)
TILE_M, TILE_N, VOX = 128, 256, 64


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


# ------------------------------------------------------------------------------------------------------------------
# geometry and the float64 reference
# ------------------------------------------------------------------------------------------------------------------
def causal_pad(k, s):
    """CausalConv3d padding (ops.ConvGeom): time at the front by (kt-1) + (1-st), space by (k-1)//2 on both sides."""
    return (k[0] - 1 + 1 - s[0], (k[1] - 1) // 2, (k[2] - 1) // 2)


def out_ext(ext, k, s, pad, strided):
    """Output grid: the input grid for a stride-1 call, else floor((in + pads - k) / s) + 1 as ops.ConvGeom.out_dims."""
    if not strided:
        return tuple(ext)
    pads = (pad[0], 2 * pad[1], 2 * pad[2])
    return tuple((e + p - kk) // ss + 1 for e, p, kk, ss in zip(ext, pads, k, s))


# ------------------------------------------------------------------------------------------------------------------
# mirror of launch_wgrad's host arithmetic (csrc/conv3d_wgrad.cu)
# ------------------------------------------------------------------------------------------------------------------
class WgradPlan:
    """The grid, the shares and the segments of one og_conv3d_wgrad* launch. Segments are (share, tile, k0, k1, slot);
    slot is None for a tile added straight into dW by its only owner. `fixup` maps each cut tile to the fixup block
    that finishes it and the slots that block adds, in order."""

    def __init__(self, sms, cout, ncols, N, out, ws_bytes, bias):
        To, Ho, Wo = out
        self.box = bw, bh, bt, bn = voxel_box(VOX, To, Ho, Wo)
        self.tiles_w, self.tiles_h, self.tiles_t = cdiv(Wo, bw), cdiv(Ho, bh), cdiv(To, bt)
        self.ksteps = cdiv(N, bn) * self.tiles_w * self.tiles_h * self.tiles_t
        self.col_tiles = cdiv(ncols, TILE_N)
        self.tiles = cdiv(cout, TILE_M) * self.col_tiles
        self.units = self.tiles * self.ksteps
        self.ctas = min(sms, max(1, self.units // 4))
        self.granule = 1
        self.slot_bytes = (TILE_M * TILE_N + (TILE_M if bias else 0)) * 4
        fit = ws_bytes // (2 * self.slot_bytes) if ws_bytes else 0
        self.path = 'stream-K'
        if fit < self.ctas:
            if fit > self.tiles:
                self.ctas, self.path = fit, 'fewer shares than SMs'
            else:
                self.granule, self.ctas, self.path = self.ksteps, min(sms, self.tiles), 'whole tiles'
        self.period = min(self.ksteps, cdiv(self.units, self.ctas))
        g = self.granule
        self.begins = [b * (self.units // g) // self.ctas * g for b in range(self.ctas + 1)]
        self.segments = []
        for b in range(self.ctas):
            u, first = self.begins[b], True
            while u < self.begins[b + 1]:
                tile = u // self.ksteps
                k0 = u - tile * self.ksteps
                k1 = min(self.ksteps, self.begins[b + 1] - tile * self.ksteps)
                whole = k0 == 0 and k1 == self.ksteps
                self.segments.append((b, tile, k0, k1, None if whole else 2 * b + (0 if first else 1)))
                u += k1 - k0
                first = False
        self.launches_fixup = self.granule == 1 and self.ctas > 1
        self.fixup = {}
        if self.launches_fixup:
            for b in range(self.ctas - 1):
                ub = self.begins[b + 1]
                tile = ub // self.ksteps
                t0, t1 = tile * self.ksteps, (tile + 1) * self.ksteps
                if ub == t0 or self.begins[b] > t0:
                    continue
                slots = []
                for sh in range(b, self.ctas):
                    sb = self.begins[sh]
                    if sb >= t1:
                        break
                    slots.append(2 * sh + (0 if sb >= t0 else 1))
                self.fixup[tile] = (b, slots)
        self.launches = 1 + int(self.launches_fixup)
        self.edge_boundaries = sum(1 for b in range(1, self.ctas) if self.begins[b] % self.ksteps == 0 and
                                   0 < self.begins[b] < self.units)

    def cut_tiles(self):
        return sorted({s[1] for s in self.segments if s[4] is not None})

    def max_segments(self):
        return max([len(v[1]) for v in self.fixup.values()] + [1])

    def describe(self):
        return (f'{self.path}: ctas {self.ctas}, granule {self.granule}, period {self.period}, tiles {self.tiles} x '
                f'{self.ksteps} k-steps, {len(self.cut_tiles())} cut tiles (up to {self.max_segments()} segments), '
                f'{self.edge_boundaries} boundaries on a tile edge, {self.launches} launch(es)')


def box_mask(plan, k, N, out):
    """Voxels of k-step k (the producer's decode in og_conv_wgrad_kernel): [N, *out] bool."""
    bw, bh, bt, bn = plan.box
    per_sample = plan.tiles_w * plan.tiles_h * plan.tiles_t
    tn, r = divmod(k, per_sample)
    tw = r % plan.tiles_w
    r //= plan.tiles_w
    th, tt = r % plan.tiles_h, r // plan.tiles_h
    m = torch.zeros((N, *out), dtype=torch.bool)
    m[tn * bn:(tn + 1) * bn, tt * bt:(tt + 1) * bt, th * bh:(th + 1) * bh, tw * bw:(tw + 1) * bw] = True
    return m


def dgrad_launches(k, s, pad, ext):
    """Implicit GEMMs og_conv3d_strided_dgrad launches: residue classes with a tap and a non-empty grid."""
    n = 0
    for cls in itertools.product(*(range(ss) for ss in s)):
        ok = True
        for d in range(3):
            r = (cls[d] - pad[d]) % s[d]
            ntap = (k[d] - 1 - cls[d]) // s[d] + 1 if cls[d] < k[d] else 0
            grid = cdiv(ext[d] - r, s[d]) if ext[d] > r else 0
            ok = ok and ntap > 0 and grid > 0
        n += ok
    return n


# ------------------------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _launches():
    from open_genie_b200 import _lib
    return _lib.launch_count()


# ------------------------------------------------------------------------------------------------------------------
# weight gradient
# ------------------------------------------------------------------------------------------------------------------
def _case(entry, cout, cin, k, N, ext, s=(1, 1, 1), pad=None, ws='scratch', ld_extra=0, off=0, n_bias=0,
          data='int', expect=None, real_cin=None, real_cout=None):
    strided = entry == 'og_conv3d_strided_wgrad'
    if pad is None:
        pad = causal_pad(k, s) if strided else tuple((kk - 1) // 2 for kk in k)
    return dict(entry=entry, cout=cout, cin=cin, k=k, s=s, pad=pad, N=N, ext=ext, ws=ws, ld_extra=ld_extra, off=off,
                n_bias=n_bias, data=data, expect=expect, real_cin=real_cin or cin, real_cout=real_cout or cout,
                out=out_ext(ext, k, s, pad, strided))


WG, WGB, WGS = 'og_conv3d_wgrad', 'og_conv3d_wgrad_bias', 'og_conv3d_strided_wgrad'
K1, K3 = (1, 1, 1), (3, 3, 3)
CAUSAL3 = (2, 1, 1)

WG_CASES = {
    # schedule paths (exact)
    'cut_one_tile': _case(WG, 128, 64, K1, 2, (16, 32, 32), expect='cut_one'),
    'cut_one_tile_bias': _case(WGB, 128, 64, K1, 2, (16, 32, 32), n_bias=128, expect='cut_one'),
    'cut_one_tile_strided': _case(WGS, 128, 64, K1, 2, (16, 64, 64), s=(1, 2, 2), pad=(0, 0, 0), expect='cut_one'),
    'many_tiles_interior': _case(WG, 256, 128, K3, 1, (5, 12, 20), expect='interior'),
    'many_tiles_interior_bias': _case(WGB, 256, 128, K3, 1, (5, 12, 20), n_bias=256, expect='interior'),
    'boundary_on_tile_edge': _case(WG, 256, 64, K1, 1, (20, 4, 16), expect='edge'),
    'boundary_on_tile_edge_bias': _case(WGB, 256, 64, K1, 1, (20, 4, 16), n_bias=200, expect='edge'),
    'fewer_shares_than_sms': _case(WG, 128, 64, K1, 2, (16, 32, 32), ws=('fit', 8), expect='fewer'),
    'fewer_shares_than_sms_bias': _case(WGB, 128, 64, K1, 2, (16, 32, 32), ws=('fit', 8), n_bias=128,
                                        expect='fewer'),
    'whole_tiles_no_workspace': _case(WG, 256, 128, K3, 1, (5, 12, 20), ws=None, expect='whole'),
    'whole_tiles_one_slot_short': _case(WG, 256, 128, K3, 1, (3, 5, 7), ws='one_short', expect='whole'),
    'whole_tiles_one_slot_short_bias': _case(WGB, 256, 128, K3, 1, (3, 5, 7), ws='one_short', n_bias=256,
                                             expect='whole'),
    'ctas_by_units': _case(WG, 72, 64, K1, 1, (5, 7, 9), expect='units'),
    'single_cta': _case(WG, 8, 64, K1, 1, (3, 5, 7), expect='single'),
    'single_cta_bias': _case(WGB, 8, 64, K1, 1, (3, 5, 7), n_bias=8, expect='single'),
    # epilogue paths (exact)
    'cout8_ncols576': _case(WG, 8, 64, (1, 3, 3), 2, (3, 9, 11)),
    'cout72_ncols384': _case(WG, 72, 128, (3, 1, 1), 2, (5, 6, 10), pad=CAUSAL3[:1] + (0, 0)),
    'cout200_ncols192': _case(WG, 200, 64, (3, 1, 1), 1, (7, 9, 5), pad=(1, 0, 0)),
    'cout256_ncols1728': _case(WG, 256, 64, K3, 1, (4, 8, 8), pad=CAUSAL3),
    'pitched_ld': _case(WG, 72, 64, K3, 1, (3, 5, 6), pad=CAUSAL3, ld_extra=40),
    'odd_ld': _case(WG, 200, 64, (1, 3, 3), 1, (3, 5, 6), ld_extra=1),
    'dw_off_8_bytes': _case(WG, 72, 128, (3, 1, 1), 1, (5, 5, 5), ld_extra=2, off=1),
    'odd_ld_strided': _case(WGS, 72, 64, K3, 1, (5, 9, 9), s=(2, 2, 2), ld_extra=3, off=1),
    'n_bias_1': _case(WGB, 72, 64, K3, 1, (3, 5, 6), n_bias=1),
    'n_bias_3_whole': _case(WGB, 64, 64, K3, 1, (3, 5, 6), n_bias=3, ws=None, expect='whole'),
    'n_bias_cout_minus_1': _case(WGB, 200, 64, K1, 2, (7, 9, 11), n_bias=199),
    'n_bias_cout_odd_ld': _case(WGB, 200, 128, (1, 3, 3), 1, (5, 6, 7), n_bias=200, ld_extra=1),
    # geometry (exact)
    'k333_causal_T1': _case(WG, 128, 64, K3, 3, (1, 6, 10), pad=CAUSAL3),
    'k333_sym_small': _case(WG, 64, 128, K3, 1, (2, 3, 3), pad=(1, 1, 1)),
    'k133_odd': _case(WG, 128, 64, (1, 3, 3), 3, (5, 7, 13)),
    'k311_causal_odd': _case(WG, 64, 64, (3, 1, 1), 5, (3, 1, 7), pad=(2, 0, 0)),
    'k111_T1_tiny': _case(WG, 64, 192, K1, 1, (1, 1, 3)),
    # strided geometry (exact)
    's122': _case(WGS, 128, 64, K3, 2, (5, 9, 11), s=(1, 2, 2)),
    's222': _case(WGS, 128, 128, K3, 2, (7, 10, 9), s=(2, 2, 2)),
    's144_k_lt_s': _case(WGS, 64, 64, K3, 2, (3, 13, 10), s=(1, 4, 4)),
    's213_nonuniform': _case(WGS, 72, 64, K3, 2, (6, 7, 13), s=(2, 1, 3)),
    's222_T2': _case(WGS, 64, 64, K3, 1, (2, 3, 3), s=(2, 2, 2)),
    # bounded, real-valued operands (n of a few thousand)
    'real_k333_causal': _case(WG, 72, 64, K3, 1, (3, 7, 9), pad=CAUSAL3, data='real'),
    'real_bias_cut': _case(WGB, 200, 64, K1, 2, (5, 9, 11), n_bias=200, data='real'),
    'real_bias_whole': _case(WGB, 128, 128, (1, 3, 3), 1, (4, 6, 9), n_bias=100, ws=None, data='real'),
    'real_strided_213': _case(WGS, 128, 64, K3, 2, (6, 7, 13), s=(2, 1, 3), data='real'),
    'real_pitched_scalar': _case(WG, 64, 128, (3, 1, 1), 1, (5, 8, 9), pad=(2, 0, 0), ld_extra=5, off=1,
                                 data='real'),
}

# Each convolution of the tokenizer (MAGVIT2 encoder / decoder, and the repr_tok stem) as ops issues its weight
# gradient: channels padded to 64 (zero input channels / zero gradient rows), n_bias = the real cout, at batch 2.
PRODUCT_CASES = {
    'enc_stem_3to128': _case(WGB, 128, 64, K3, 2, (4, 8, 8), pad=CAUSAL3, n_bias=128, real_cin=3),
    'res_conv_128to128': _case(WG, 128, 128, K3, 2, (4, 8, 8), pad=(1, 1, 1)),
    'res_conv_128to256': _case(WG, 256, 128, K3, 2, (4, 8, 8), pad=(1, 1, 1)),
    'res_conv_256to512': _case(WG, 512, 256, K3, 2, (2, 4, 4), pad=(1, 1, 1)),
    'res_conv_512to512': _case(WG, 512, 512, K3, 2, (2, 4, 4), pad=(1, 1, 1)),
    'shortcut_128to256': _case(WGB, 256, 128, K1, 2, (4, 8, 8), n_bias=256),
    'shortcut_256to512': _case(WGB, 512, 256, K1, 2, (2, 4, 4), n_bias=512),
    'down_122_128': _case(WGS, 128, 128, K3, 2, (4, 16, 16), s=(1, 2, 2)),
    'down_222_256': _case(WGS, 256, 256, K3, 2, (4, 8, 8), s=(2, 2, 2)),
    'enc_out_512to18': _case(WGB, 64, 512, K1, 2, (2, 4, 4), n_bias=18, real_cout=18),
    'dec_stem_18to512': _case(WGB, 512, 64, K3, 2, (2, 4, 4), pad=CAUSAL3, n_bias=512, real_cin=18),
    'up_512to4096': _case(WGB, 4096, 512, K3, 1, (2, 4, 4), pad=CAUSAL3, n_bias=4096),
    'up_256to2048': _case(WGB, 2048, 256, K3, 2, (2, 4, 4), pad=CAUSAL3, n_bias=2048),
    'up_256to1024': _case(WGB, 1024, 256, K3, 2, (4, 8, 8), pad=CAUSAL3, n_bias=1024),
    'dec_out_128to3': _case(WGB, 64, 128, K3, 2, (4, 8, 8), pad=CAUSAL3, n_bias=3, real_cout=3),
    'repr_stem_144_3to512': _case(WGS, 512, 64, K3, 2, (2, 16, 16), s=(1, 4, 4), real_cin=3),
}


def ws_bytes_of(c, sms):
    ws = c['ws']
    if ws is None:
        return 0
    if ws == 'scratch':
        return SCRATCH
    bias = c['entry'] == WGB
    full = WgradPlan(sms, c['cout'], _ncols(c), c['N'], c['out'], SCRATCH, bias)
    slot = full.slot_bytes
    if ws == 'one_short':
        return (2 * full.ctas - 1) * slot
    return 2 * slot * ws[1]


def _ncols(c):
    return math.prod(c['k']) * c['cin']


def plan_of(c, sms):
    return WgradPlan(sms, c['cout'], _ncols(c), c['N'], c['out'], ws_bytes_of(c, sms), c['entry'] == WGB)


def assert_path(plan, expect, sms):
    """The schedule path a case exists for is the one the mirror says it takes on this SM count."""
    d = plan.describe()
    if expect == 'cut_one':
        assert plan.tiles == 1 and plan.max_segments() == plan.ctas == min(sms, plan.units // 4), d
    elif expect == 'interior':
        assert plan.path == 'stream-K' and len(plan.cut_tiles()) > 1 and plan.tiles > 1, d
    elif expect == 'edge':
        assert plan.path == 'stream-K' and plan.edge_boundaries > 0 and plan.fixup, d
    elif expect == 'fewer':
        assert plan.path == 'fewer shares than SMs' and plan.tiles < plan.ctas < sms and plan.fixup, d
    elif expect == 'whole':
        assert plan.path == 'whole tiles' and plan.launches == 1 and not plan.cut_tiles(), d
    elif expect == 'units':
        assert plan.ctas == plan.units // 4 < sms and plan.ctas > 1, d
    elif expect == 'single':
        assert plan.ctas == 1 and plan.launches == 1, d


def wgrad_inputs(c, seed, device=DEV):
    N, (T, H, W), (To, Ho, Wo) = c['N'], c['ext'], c['out']
    x = operand((N, T, H, W, c['cin']), seed, c['data'], device)
    dy = operand((N, To, Ho, Wo, c['cout']), seed + 1, c['data'], device)
    x[..., c['real_cin']:] = 0         # channel padding of the narrow stems
    dy[..., c['real_cout']:] = 0       # zero gradient rows of a padded cout
    init_kind = c['data']
    dw0 = operand((c['cout'], _ncols(c)), seed + 2, init_kind, device, F32T, -5, 5)
    db0 = operand((c['cout'],), seed + 3, init_kind, device, F32T, -5, 5)
    return x, dy, dw0, db0


def wgrad_run(c, x, dy, dw0, db0, sms):
    """One call on guarded, NaN-filled dW / db / workspace. Returns dW [cout, ncols], db [n_bias] and the launches."""
    cout, cin, ncols, n_bias = c['cout'], c['cin'], _ncols(c), c['n_bias']
    ld = ncols + c['ld_extra']
    dwg = Guarded((cout, ld), F32T, offset=c['off'])
    dwg.t[:, :ncols].copy_(dw0)
    dbg = Guarded((cout,), F32T)
    dbg.t[:n_bias].copy_(db0[:n_bias])
    wsb = ws_bytes_of(c, sms)
    wsg = Guarded((max(wsb // 4, 1),), F32T)
    ws = (wsg.ptr(), wsb) if wsb else (None, 0)
    N, (T, H, W), k, pad, s = c['N'], c['ext'], c['k'], c['pad'], c['s']
    n0 = _launches()
    if c['entry'] == WGS:
        _call(WGS, dy.data_ptr(), cout, x.data_ptr(), cin, dwg.ptr(), ld, *k, *s, *pad, N, T, H, W, *ws)
    elif c['entry'] == WGB:
        _call(WGB, dy.data_ptr(), cout, x.data_ptr(), cin, dwg.ptr(), ld, *k, *pad, N, T, H, W, dbg.ptr(), n_bias, *ws)
    else:
        _call(WG, dy.data_ptr(), cout, x.data_ptr(), cin, dwg.ptr(), ld, *k, *pad, N, T, H, W, *ws)
    torch.cuda.synchronize()
    launches = _launches() - n0
    dwg.check_guard('dW')
    dbg.check_guard('db')
    wsg.check_guard('workspace')
    assert _nan_bits(dwg.t[:, ncols:]), 'dW: the words between rows were written'
    assert _nan_bits(dbg.t[n_bias:]), 'db: entries past n_bias were written'
    if c['entry'] != WGB:
        assert dbg.untouched(), 'db written by an entry point without a bias'
    return dwg.t[:, :ncols].clone(), dbg.t[:n_bias].clone(), launches


def wgrad_expect(c, x, dy, dw0, db0, plan):
    """(reference, bound) for dW and db; exact cases get a zero bound after checking they are exact."""
    k, s, pad, cout, cin = c['k'], c['s'], c['pad'], c['cout'], c['cin']
    xd, dyd = x.double(), dy.double()
    ref_w = wgrad_ref(xd, dyd, k, s, pad).reshape(cout, -1) + dw0.double()
    mag_w = wgrad_ref(xd.abs(), dyd.abs(), k, s, pad).reshape(cout, -1) + dw0.double().abs()
    ref_b = dyd.reshape(-1, cout).sum(0) + db0.double()
    mag_b = dyd.abs().reshape(-1, cout).sum(0) + db0.double().abs()
    if c['data'] == 'int':
        assert mag_w.max() <= EXACT_LIMIT and mag_b.max() <= EXACT_LIMIT, 'case too large for the exact check'
        return ref_w, 0.0, ref_b, 0.0
    n = c['N'] * math.prod(c['out']) + plan.max_segments() + 1
    return ref_w, gam(n) * SLACK * mag_w, ref_b, gam(n) * SLACK * mag_b


def wgrad_case(name, c):
    sms = num_sms()
    plan = plan_of(c, sms)
    if c['expect']:
        assert_path(plan, c['expect'], sms)
    print(f'{name} ({sms} SMs): {plan.describe()}')
    x, dy, dw0, db0 = wgrad_inputs(c, zlib.crc32(name.encode()))
    dw, db, launches = wgrad_run(c, x, dy, dw0, db0, sms)
    assert launches == plan.launches, (name, launches, plan.describe())
    ref_w, tol_w, ref_b, tol_b = wgrad_expect(c, x, dy, dw0, db0, plan)
    check(f'{name} dW', dw, ref_w, tol_w)
    if c['entry'] == WGB:
        check(f'{name} db', db, ref_b[:c['n_bias']], tol_b if isinstance(tol_b, float) else tol_b[:c['n_bias']])
    dw2, db2, _ = wgrad_run(c, x, dy, dw0, db0, sms)
    assert torch.equal(dw.view(torch.int32), dw2.view(torch.int32)), f'{name}: dW differs between two runs'
    assert torch.equal(db.view(torch.int32), db2.view(torch.int32)), f'{name}: db differs between two runs'


@GPU
@pytest.mark.parametrize('name', list(WG_CASES))
def test_wgrad_paths(name):
    wgrad_case(name, WG_CASES[name])


@GPU
@pytest.mark.parametrize('name', list(PRODUCT_CASES))
def test_wgrad_product_geometry(name):
    wgrad_case(name, PRODUCT_CASES[name])


# ------------------------------------------------------------------------------------------------------------------
# strided forward and data gradient
# ------------------------------------------------------------------------------------------------------------------
STRIDED_GEOMS = [  # (kernel, stride, input extents): partial boxes, odd extents, k < s, a non-uniform stride
    (K3, (1, 2, 2), (5, 9, 11)),
    (K3, (2, 2, 2), (7, 10, 9)),
    (K3, (1, 4, 4), (3, 13, 10)),
    (K3, (2, 1, 3), (6, 7, 13)),
]


def _strided_w(cout, k, cin, ldw, seed, kind, w_rows=None):
    """bf16 weights [cout][ldw]: the ntaps*cin real columns, NaN in the pitch columns and in the rows from w_rows on
    (none of which may be read)."""
    wg = Guarded((cout, ldw), BF16)
    ntk = math.prod(k) * cin
    rows = cout if w_rows is None else w_rows
    wg.t[:rows, :ntk].copy_(operand((rows, ntk), seed, kind))
    return wg


FWD_CASES = {f'cout{co}_{"f32" if f32 else "bf16"}{"_bias" if b else ""}': (co, f32, b, i)
             for i, (co, f32, b) in enumerate(itertools.product((18, 64, 128, 192, 512), (0, 1), (0, 1)))}


def fwd_case(name, cout, out_f32, has_bias, geom_i, kind='int'):
    k, s, ext = STRIDED_GEOMS[geom_i % len(STRIDED_GEOMS)]
    cin, N = (64, 128)[geom_i % 2], 2
    pad = causal_pad(k, s)
    out = out_ext(ext, k, s, pad, True)
    seed = zlib.crc32(name.encode())
    x = operand((N, *ext, cin), seed, kind)
    ntk = math.prod(k) * cin
    ldw = ntk + 8
    wg = _strided_w(cout, k, cin, ldw, seed + 1, kind)
    bias = operand((cout,), seed + 2, kind, dtype=F32T, lo=-20, hi=20) if has_bias else None
    odt = F32T if out_f32 else BF16
    runs = []
    for _ in range(2):
        og = Guarded((N, *out, cout), odt)
        n0 = _launches()
        _call('og_conv3d_strided_fwd', x.data_ptr(), cin, *k, *s, *pad, wg.ptr(), ldw,
              None if bias is None else bias.data_ptr(), og.ptr(), out_f32, N, *ext, cout)
        torch.cuda.synchronize()
        assert _launches() - n0 == 1
        og.check_guard('out')
        runs.append(og.t.clone())
    ity = Guarded.BITS[odt][0]
    assert torch.equal(runs[0].view(ity), runs[1].view(ity)), f'{name}: two runs differ'
    w3 = wg.t[:, :ntk].double().view(cout, -1, cin)
    ref = fwd_ref(x.double(), w3, k, s, pad, out)
    mag = fwd_ref(x.double().abs(), w3.abs(), k, s, pad, out)
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    if kind == 'int':
        assert mag.max() <= EXACT_LIMIT
        want = ref if out_f32 else ref.to(BF16)
        check_exact(name, runs[0], want)
    else:
        err = gam(ntk + 1) * SLACK * mag
        tol = err if out_f32 else (1 + U) * err + U * ref.abs()
        check(name, runs[0], ref, tol)


@GPU
@pytest.mark.parametrize('name', list(FWD_CASES))
def test_strided_fwd(name):
    fwd_case(name, *FWD_CASES[name])


@GPU
@pytest.mark.parametrize('cout,out_f32', [(64, 0), (192, 1)])
def test_strided_fwd_real(cout, out_f32):
    for i in range(len(STRIDED_GEOMS)):
        fwd_case(f'real_cout{cout}_geom{i}', cout, out_f32, True, i, kind='real')


DGRAD_CASES = {   # (geometry index, input extents or None for the geometry's own, cout, w_rows, cin, data)
    'g0': (0, None, 64, 64, 64, 'int'),
    'g1_wrows18': (1, None, 64, 18, 128, 'int'),
    'g2_k_lt_s': (2, None, 128, 128, 64, 'int'),
    'g2_k_lt_s_wrows100': (2, (2, 9, 7), 128, 100, 64, 'int'),
    'g3_nonuniform': (3, None, 64, 64, 64, 'int'),
    'g3_empty_classes': (3, (2, 2, 2), 64, 3, 128, 'int'),     # extents below the stride: classes with no grid
    'g2_empty_classes': (2, (1, 3, 2), 64, 64, 64, 'int'),
    'g0_T1': (0, (1, 4, 5), 64, 64, 64, 'int'),
    'g1_T2': (1, (2, 4, 5), 64, 64, 64, 'int'),
    'real_g1': (1, None, 64, 50, 64, 'real'),
    'real_g3': (3, None, 128, 128, 128, 'real'),
}


def unreached_rows(k, s, pad, ext):
    """[T, H, W] bool: input positions whose residue class has no tap (k < s), which must be exactly +0."""
    ms = []
    for d in range(3):
        cls = (torch.arange(ext[d]) + pad[d]) % s[d]
        ms.append(cls >= k[d])
    return ms[0][:, None, None] | ms[1][None, :, None] | ms[2][None, None, :]


@GPU
@pytest.mark.parametrize('name', list(DGRAD_CASES))
def test_strided_dgrad(name):
    gi, ext, cout, w_rows, cin, kind = DGRAD_CASES[name]
    k, s, ext0 = STRIDED_GEOMS[gi]
    ext = ext or ext0
    pad = causal_pad(k, s)
    out = out_ext(ext, k, s, pad, True)
    N = 2
    seed = zlib.crc32(name.encode())
    dy = operand((N, *out, cout), seed, kind)
    dy[..., w_rows:] = 0                       # the caller zero-pads dy's channels past the real weight rows
    ntk = math.prod(k) * cin
    ldw = ntk + 16
    wg = _strided_w(cout, k, cin, ldw, seed + 1, kind, w_rows)
    runs = []
    for _ in range(2):
        dxg = Guarded((N, *ext, cin), BF16)
        n0 = _launches()
        _call('og_conv3d_strided_dgrad', dy.data_ptr(), cout, w_rows, wg.ptr(), ldw, *k, *s, *pad, dxg.ptr(), N, *ext,
              cin)
        torch.cuda.synchronize()
        assert _launches() - n0 == dgrad_launches(k, s, pad, ext), name
        dxg.check_guard('dx')
        runs.append(dxg.t.clone())
    assert torch.equal(runs[0].view(torch.int16), runs[1].view(torch.int16)), f'{name}: two runs differ'
    dx = runs[0]
    w3 = wg.t[:w_rows, :ntk].double().view(w_rows, -1, cin)
    dyd = dy[..., :w_rows].double()
    ref = dgrad_ref(dyd, w3, k, s, pad, ext)
    mag = dgrad_ref(dyd.abs(), w3.abs(), k, s, pad, ext)
    zero = unreached_rows(k, s, pad, ext).to(DEV)
    if zero.any():
        z = dx[:, zero]
        assert (z.view(torch.int16) == 0).all(), f'{name}: rows no tap reaches are not +0'
    if kind == 'int':
        assert mag.max() <= EXACT_LIMIT
        check_exact(name, dx, ref.to(BF16))
    else:
        err = gam(math.prod(k) * w_rows) * SLACK * mag
        check(name, dx, ref, (1 + U) * err + U * ref.abs())


@GPU
def test_downsample_rejects_input_shorter_than_kernel():
    """T = 1 into a time-stride-2 causal downsample (kt = 3, pt = 1) has no output frame, as in F.conv3d."""
    from open_genie_b200.module.video import SpaceTimeDownsample
    m = SpaceTimeDownsample(64, 3, time_factor=2, space_factor=2).to(DEV)
    x = torch.randn(1, 64, 1, 8, 8, device=DEV)
    with pytest.raises(ValueError, match='smaller than the kernel'):
        m(x)
    assert tuple(m(torch.randn(1, 64, 2, 8, 8, device=DEV)).shape) == (1, 64, 1, 4, 4)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference against torch
# ------------------------------------------------------------------------------------------------------------------
def _ref_geometries():
    g = set()
    for cases, strided_entry in ((WG_CASES, WGS), (PRODUCT_CASES, WGS)):
        for c in cases.values():
            g.add((c['k'], c['s'], c['pad'], c['entry'] == strided_entry))
    for k, s, _ in STRIDED_GEOMS:
        g.add((k, s, causal_pad(k, s), True))
    return sorted(g)


@pytest.mark.parametrize('geom', _ref_geometries(), ids=str)
def test_reference_matches_torch(geom):
    k, s, pad, strided = geom
    for ext in ((1, 3, 2), (5, 7, 9), (4, 8, 8)):
        out = out_ext(ext, k, s, pad, strided)
        if min(out) < 1:
            continue
        x = operand((2, *ext, 5), 11, 'real', 'cpu', F64T)
        w = operand((3, math.prod(k), 5), 12, 'real', 'cpu', F64T)
        dy = operand((2, *out, 3), 13, 'real', 'cpu', F64T)
        for op, mine in (('fwd', fwd_ref(x, w, k, s, pad, out)), ('wgrad', wgrad_ref(x, dy, k, s, pad)),
                         ('dgrad', dgrad_ref(dy, w, k, s, pad, ext))):
            ref = torch_ref(op, x, w, dy, k, s, pad, ext)
            assert mine.shape == ref.shape, (op, ext, mine.shape, ref.shape)
            # float64 sums in another order: relative to the largest term (operands span 2^-10 .. 2^10)
            err = float((mine - ref).abs().max())
            assert err <= 1e-12 * float(ref.abs().max()), (op, geom, ext, err)


def test_out_dims_rejects_input_shorter_than_kernel():
    from open_genie_b200 import ops
    g = ops.ConvGeom(64, 64, K3, (2, 2, 2))
    assert g.pt == 1 and g.out_dims(2, 8, 8) == (1, 4, 4)
    with pytest.raises(ValueError, match='smaller than the kernel'):
        g.out_dims(1, 8, 8)
    with pytest.raises(RuntimeError):
        F.conv3d(F.pad(torch.zeros(1, 1, 1, 8, 8), (1, 1, 1, 1, 1, 0)), torch.zeros(1, 1, 3, 3, 3), stride=2)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the schedule mirror
# ------------------------------------------------------------------------------------------------------------------
def check_plan_invariants(p, ws_bytes):
    assert p.begins[0] == 0 and p.begins[-1] == p.units
    assert all(a <= b for a, b in zip(p.begins, p.begins[1:]))
    assert all(b % p.granule == 0 for b in p.begins)
    covered = 0
    by_share, by_tile = {}, {}
    for share, tile, k0, k1, slot in p.segments:
        assert 0 <= k0 < k1 <= p.ksteps
        covered += k1 - k0
        by_share.setdefault(share, []).append(slot)
        by_tile.setdefault(tile, []).append((k0, k1, slot))
    assert covered == p.units
    for slots in by_share.values():          # a share leaves at most two cut segments, in distinct slots
        cut = [sl for sl in slots if sl is not None]
        assert len(cut) <= 2 and len(set(cut)) == len(cut)
    cut_tiles = p.cut_tiles()
    assert sorted(p.fixup) == cut_tiles       # every cut tile is finished by exactly one fixup block
    for tile in cut_tiles:
        segs = sorted(by_tile[tile])
        assert segs[0][0] == 0 and segs[-1][1] == p.ksteps
        assert all(a[1] == b[0] for a, b in zip(segs, segs[1:]))
        slots = [sl for _, _, sl in segs]
        assert None not in slots
        assert p.fixup[tile][1] == slots, (tile, p.fixup[tile], slots)   # the fixup adds them in k order
        assert len(set(slots)) == len(slots)
    used = [s[4] for s in p.segments if s[4] is not None]
    if used:
        assert p.launches_fixup and max(used) < 2 * p.ctas and 2 * p.ctas * p.slot_bytes <= ws_bytes
    else:
        assert not p.fixup
    assert p.launches == 1 + int(p.granule == 1 and p.ctas > 1)
    assert 1 <= p.period <= p.ksteps


@pytest.mark.parametrize('sms', [1, 7, 16, 114, 132])
def test_wgrad_plan_invariants(sms):
    shapes = [(c['cout'], _ncols(c), c['N'], c['out']) for c in list(WG_CASES.values()) + list(PRODUCT_CASES.values())]
    shapes += [(cout, ncols, N, (T, H, W)) for cout in (8, 128, 200, 512) for ncols in (64, 576, 1728, 6912)
               for N, T, H, W in ((1, 1, 1, 1), (2, 5, 7, 9), (8, 16, 32, 32), (1, 3, 64, 64))]
    slot = TILE_M * TILE_N * 4
    for cout, ncols, N, out in shapes:
        for bias in (False, True):
            for ws in (0, SCRATCH, 2 * slot, 2 * (slot + 512) * 5, 2 * (slot + 512) * 40 - 1, 1 << 20):
                p = WgradPlan(sms, cout, ncols, N, out, ws, bias)
                check_plan_invariants(p, ws)


def test_wgrad_cases_reach_their_paths_on_common_sm_counts():
    for sms in (114, 132):
        for name, c in WG_CASES.items():
            if c['expect']:
                assert_path(plan_of(c, sms), c['expect'], sms)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the checks reject the mistakes they exist for
# ------------------------------------------------------------------------------------------------------------------
SENS = _case(WGB, 128, 64, (3, 3, 3), 2, (5, 6, 7), pad=CAUSAL3, n_bias=128, data='real')
SENS_STRIDED = _case(WGS, 64, 64, (3, 3, 3), 2, (5, 8, 9), s=(2, 2, 2), data='real')


def _wgrad_mistakes(c, x, dy, plan):
    """dW / db as the kernel would produce them with each mistake (float64, before the initial value)."""
    k, s, pad, cout = c['k'], c['s'], c['pad'], c['cout']
    N, out = c['N'], c['out']
    ref = wgrad_ref(x, dy, k, s, pad).reshape(cout, -1)

    def partial(kset):     # dW of the given k-steps only
        m = torch.zeros((N, *out), dtype=torch.bool)
        for kk in kset:
            m |= box_mask(plan, kk, N, out)
        return wgrad_ref(x, dy * m[..., None], k, s, pad).reshape(cout, -1)
    tile = (slice(0, min(cout, TILE_M)), slice(0, min(_ncols(c), TILE_N)))
    dropped = ref.clone()
    dropped[tile] -= partial([plan.ksteps - 1])[tile]     # the last box: every tap reaches inside x there
    doubled = ref.clone()
    doubled[tile] += partial(range(0, max(1, plan.ksteps // 3)))[tile]
    xh = x.to(BF16).view(torch.float16).double() if x.dtype != BF16 else x.view(torch.float16).double()
    fp16 = wgrad_ref(torch.nan_to_num(xh, posinf=6e4, neginf=-6e4), dy, k, s, pad).reshape(cout, -1)
    out = {
        'one 64-voxel box dropped from one tile': dropped,
        'a cut segment added twice': doubled,
        'taps mirrored': wgrad_ref(x, dy, k, s, pad, ('mirror',)).reshape(cout, -1),
        'stride offset by one': wgrad_ref(x, dy, k, s, pad, ('stride_off',)).reshape(cout, -1),
        'bf16 operand read as fp16': fp16,
    }
    if pad[0] != (k[0] - 1) // 2:
        out['causal padding applied symmetrically'] = wgrad_ref(x, dy, k, s, pad, ('causal_sym',)).reshape(cout, -1)
    return ref, out


@pytest.mark.parametrize('c', [SENS, SENS_STRIDED], ids=['stride1', 'strided'])
def test_bounds_reject_wgrad_mistakes(c):
    plan = WgradPlan(132, c['cout'], _ncols(c), c['N'], c['out'], SCRATCH, c['entry'] == WGB)
    x, dy, dw0, db0 = wgrad_inputs(c, 7, 'cpu')
    ref_w, tol_w, ref_b, tol_b = wgrad_expect(c, x, dy, dw0, db0, plan)
    assert float(tol_w.max()) > 0
    xd, dyd = x.double(), dy.double()
    exact, mistakes = _wgrad_mistakes(c, xd, dyd, plan)
    check('correct', exact + dw0.double(), ref_w, tol_w)
    assert len(mistakes) >= 5
    for what, got in mistakes.items():
        _rejects(lambda: check(what, got + dw0.double(), ref_w, tol_w))
    if c['entry'] == WGB:
        wrong_rows = dyd.reshape(-1, c['cout']).roll(1, dims=1).sum(0) + db0.double()
        check('db', dyd.reshape(-1, c['cout']).sum(0) + db0.double(), ref_b, tol_b)
        _rejects(lambda: check('bias summed over the wrong rows', wrong_rows, ref_b, tol_b))
    # integer data: every mistake changes at least one element, so the exact check fails too
    ci = dict(c, data='int')
    xi, dyi, _, _ = wgrad_inputs(ci, 8, 'cpu')
    ref_i, mistakes_i = _wgrad_mistakes(ci, xi.double(), dyi.double(), plan)
    for what, got in mistakes_i.items():
        assert not torch.equal(got, ref_i), f'integer data does not see: {what}'
    wrong_rows = dyi.double().reshape(-1, c['cout']).roll(1, dims=1).sum(0)
    assert not torch.equal(wrong_rows, dyi.double().reshape(-1, c['cout']).sum(0))


def test_bounds_reject_strided_fwd_and_dgrad_mistakes():
    k, s, ext = K3, (1, 2, 2), (5, 8, 9)
    pad = causal_pad(k, s)
    out = out_ext(ext, k, s, pad, True)
    x = operand((2, *ext, 64), 21, 'real', 'cpu').double()
    w = operand((64, 27, 64), 22, 'real', 'cpu').double()
    dy = operand((2, *out, 64), 23, 'real', 'cpu').double()
    y = fwd_ref(x, w, k, s, pad, out)
    tol_y = (1 + U) * gam(27 * 64 + 1) * SLACK * fwd_ref(x.abs(), w.abs(), k, s, pad, out) + U * y.abs()
    check('fwd', y.to(BF16), y, tol_y)
    dx = dgrad_ref(dy, w, k, s, pad, ext)
    tol_x = (1 + U) * gam(27 * 64) * SLACK * dgrad_ref(dy.abs(), w.abs(), k, s, pad, ext) + U * dx.abs()
    check('dgrad', dx.to(BF16), dx, tol_x)
    for mut in (('mirror',), ('stride_off',), ('causal_sym',)):
        _rejects(lambda: check(f'fwd {mut}', fwd_ref(x, w, k, s, pad, out, mut), y, tol_y))
        _rejects(lambda: check(f'dgrad {mut}', dgrad_ref(dy, w, k, s, pad, ext, mut), dx, tol_x))
    xh = x.to(BF16).view(torch.float16).double()
    _rejects(lambda: check('fwd fp16', fwd_ref(torch.nan_to_num(xh), w, k, s, pad, out), y, tol_y))
    # a weight row past w_rows read (its NaN would spread) or a tap class stored at the wrong offset
    _rejects(lambda: check('dgrad shifted class', dx.roll(1, dims=2), dx, tol_x))


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation (host buffers, no CUDA call)
# ------------------------------------------------------------------------------------------------------------------
def test_conv_argument_validation_returns_status_codes():
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    p = (ctypes.addressof(buf) + 255) & ~255

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error(), text)

    def wg(cout=64, cin=64, ld=27 * 64, k=K3, pad=CAUSAL3, N=1, T=4, H=8, W=8, dw=p):
        return lib.og_conv3d_wgrad(p, cout, p, cin, dw, ld, *k, *pad, N, T, H, W, None, 0, None)

    def wb(cout=64, n_bias=64, db=p):
        return lib.og_conv3d_wgrad_bias(p, cout, p, 64, p, 27 * 64, *K3, *CAUSAL3, 1, 4, 8, 8, db, n_bias, None, 0,
                                         None)

    def sw(cout=64, cin=64, ld=27 * 64, k=K3, s=(2, 2, 2), pad=(1, 1, 1), N=1, T=4, H=8, W=8):
        return lib.og_conv3d_strided_wgrad(p, cout, p, cin, p, ld, *k, *s, *pad, N, T, H, W, None, 0, None)

    def sf(cin=64, k=K3, s=(2, 2, 2), pad=(1, 1, 1), ldw=27 * 64, N=1, T=4, H=8, W=8, cout=64):
        return lib.og_conv3d_strided_fwd(p, cin, *k, *s, *pad, p, ldw, None, p, 0, N, T, H, W, cout, None)

    def sd(cout=64, w_rows=64, ldw=27 * 64, k=K3, s=(2, 2, 2), pad=(1, 1, 1), N=1, T=4, H=8, W=8, cin=64):
        return lib.og_conv3d_strided_dgrad(p, cout, w_rows, p, ldw, *k, *s, *pad, p, N, T, H, W, cin, None)

    # 1. a dW row stride below kt*kh*kw*cin (rows would overlap)
    bad(wg(ld=27 * 64 - 8), b'ld_dw=1720 must be >= kt*kh*kw*cin = 1728')
    bad(wg(ld=0), b'ld_dw')
    bad(sw(ld=27 * 64 - 1), b'ld_dw')
    # 2. non-positive extents
    for N, T, H, W_ in ((0, 4, 8, 8), (1, 0, 8, 8), (1, 4, -1, 8), (1, 4, 8, 0)):
        bad(wg(N=N, T=T, H=H, W=W_), b'extents must be positive')
        bad(sf(N=N, T=T, H=H, W=W_), b'conv3d_strided_fwd')
        bad(sd(N=N, T=T, H=H, W=W_), b'conv3d_strided_dgrad')
    bad(sw(N=0), b'extents must be positive')
    # 3. a padded extent smaller than the kernel: T = 1, kt = 3, pt = 1, st = 2 has no output frame
    bad(sw(T=1), b'smaller than the kernel')
    bad(sf(T=1), b'empty output')
    bad(sd(T=1), b'empty output')
    bad(sf(H=1, pad=(1, 0, 1)), b'empty output')
    bad(sw(W=2, pad=(1, 1, 0), s=(2, 2, 1)), b'smaller than the kernel')
    # stride 0 (used to divide by zero on the host) and the strided data gradient's ldw
    bad(sw(s=(0, 2, 2)), b'bad stride')
    bad(sd(s=(2, 0, 2)), b'bad kernel / stride / padding')
    bad(sd(ldw=27 * 64 - 8), b'bad w_rows / ldw')
    # the checks that already existed
    bad(wg(dw=None), b'null pointer')
    bad(lib.og_conv3d_wgrad_bias(p, 64, p, 64, p, 27 * 64, *K3, *CAUSAL3, 1, 4, 8, 8, None, 64, None, 0, None),
        b'dbias is NULL')
    for n_bias in (0, -1, 65):
        bad(wb(n_bias=n_bias), b'n_bias')
    bad(wg(cin=96, ld=27 * 96), b'cin=96 must be a multiple of 64')
    bad(wg(cout=12), b'cout=12 must be a multiple of 8')
    bad(wg(pad=(3, 1, 1)), b'bad kernel/padding')
    bad(wg(pad=(0, 1, -1)), b'bad kernel/padding')
    bad(sw(s=(9, 1, 1), pad=(0, 1, 1), T=20), b'bad stride')
    bad(sf(s=(1, 9, 1), pad=(2, 1, 1)), b'bad kernel / stride / padding')
    bad(sd(s=(1, 1, 9), pad=(2, 1, 1)), b'bad kernel / stride / padding')
    bad(sd(cout=72), b'multiples of 64')
    bad(sd(w_rows=65), b'bad w_rows / ldw')
    bad(sf(ldw=27 * 64 - 8), b'bad ldw')
    # strided boxes wider than 256 input positions (x: 64 output columns x stride 8; forward: 128 x 3)
    bad(sw(k=K1, s=(1, 1, 8), pad=(0, 0, 0), ld=64, T=1, H=1, W=257), b'strided box exceeds the TMA limit')
    bad(sf(k=K1, s=(1, 1, 3), pad=(0, 0, 0), ldw=64, T=1, H=1, W=384), b'strided box exceeds the TMA limit')
