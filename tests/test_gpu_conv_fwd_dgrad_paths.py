"""Every path of the stride-1 convolution forward and data gradient (og_conv3d_fwd, og_conv3d_dgrad) through the C ABI,
against the float64 "convolution by taps" reference of conv_ref.py.

Two kinds of check, as in test_gpu_conv_wgrad_strided_paths.py:
- Exact. x, dy, w, the biases and the residual are small integers and every output element's sum of |terms| stays
  below 2^22, so every partial sum, in any order and any split, is an integer fp32 holds exactly. fp32 outputs must
  EQUAL the float64 reference and bf16 outputs its single rounding to bf16. Some cases reach magnitudes above 256, so
  that the bf16 rounding really rounds (a residual added after it then changes the result). The GroupNorm sums must
  equal the float64 sums of the kernel's own bf16 output: per sample, the sum of |y| and of y^2 stays below 2^24, which
  bounds every fp32 partial any sums path forms (per row and per 32 rows in the fused epilogues, per thread and per
  block in the split-K finish pass, per thread in og_gn_stats).
- Bounded. Real operands with exponents spread over 2^+-10 and random signs, and per-element bounds gam(n) * sum|terms|
  (+ U * |ref| for bf16 outputs). These catch type and descriptor errors that integer data cannot.

Every output sits in a NaN-filled `Guarded` buffer; the weights' pitch columns and their rows from w_rows on are NaN,
so reading one shows; every case runs twice and must give the same bits.

`IgemmPlan` mirrors launch_igemm's host arithmetic (csrc/conv3d_igemm.cu): which kernel instantiation, tile, split,
store and GroupNorm-sums path a call takes for a given SM count, and how many kernels it launches. Every GPU case checks
the launch count against it, and a profiler test checks the kernel names once per path. CPU tests check that every
case reaches its path at 114 and 132 SMs (H100 PCIe and SXM), the mirror's invariants, the reference against torch, that
the bounds and the integer data reject the mistakes they exist for, and that bad arguments return -1 before any CUDA
call.
"""
import ctypes
import math
import re
import zlib

import pytest
import torch

from conv_ref import (BF16, DEV, EXACT_LIMIT, F32T, F64T, SLACK, U, cdiv, check, dgrad_ref, fwd_ref, gam, nan_bits,
                      operand, rejects, torch_ref, voxel_box)
from helpers import Guarded

GPU = pytest.mark.gpu
WS_FULL = 24 << 20          # the step scope's split-K workspace (ops.StepScope.workspace)
TILE_M, SWAP_VOX, WIDE_N = 128, 256, 256
SUM_LIMIT = 2 ** 24         # per sample: sum |y| and sum y^2 of the exact GroupNorm-sums cases
ONE = (1, 1, 1)


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


# ------------------------------------------------------------------------------------------------------------------
# mirror of launch_igemm's host arithmetic (csrc/conv3d_igemm.cu)
# ------------------------------------------------------------------------------------------------------------------
def pick_block_n(n_out, mn_major):
    bn = 16
    while bn < n_out and bn < 128:
        bn *= 2
    return max(bn, 64) if mn_major else bn


class IgemmPlan:
    """One og_conv3d_fwd / og_conv3d_dgrad call on `sms` SMs. c0 is the K segment's channel count (x0's for the
    forward, dy's for the data gradient), n_out the output channels."""

    def __init__(self, sms, dgrad, c0, k, N, ext, n_out, c1=0, out_f32=False, residual=False, ws_bytes=0,
                 sums=False):
        T, H, W = ext
        vox = N * T * H * W
        self.swap = not out_f32 and not residual and n_out == 128 and vox >= 4 * SWAP_VOX * sms
        self.box = bw, bh, bt, bn = voxel_box(SWAP_VOX if self.swap else TILE_M, T, H, W)
        self.partial = ''.join(a for a, e, b in zip('wht', (W, H, T), (bw, bh, bt)) if e % b)
        self.num_kb = c0 // 64 * math.prod(k) + c1 // 64
        self.m_tiles = cdiv(N, bn) * cdiv(W, bw) * cdiv(H, bh) * cdiv(T, bt)
        self.block_n = pick_block_n(n_out, dgrad)
        self.n_tiles = cdiv(n_out, self.block_n)
        self.vec_ok = n_out % (4 if out_f32 else 8) == 0
        self.fast_store = not out_f32 and n_out % 64 == 0 and self.block_n % 64 == 0
        self.slab = vox * n_out * 4
        self.splits = 1
        tiles = self.m_tiles * self.n_tiles
        if tiles * 2 <= sms and self.num_kb >= 32 and ws_bytes and not residual:
            sp = min(sms // tiles, self.num_kb // 8, 16, ws_bytes // self.slab)
            if sp >= 2:
                self.splits = sp
        self.wide = (self.splits == 1 and self.fast_store and n_out >= WIDE_N and
                     (not dgrad or (n_out == WIDE_N and c0 <= 1024)))
        if self.wide:
            self.block_n, self.n_tiles = WIDE_N, cdiv(n_out, WIDE_N)
        self.items = self.m_tiles * self.n_tiles * self.splits
        self.grid = min(sms, self.items)
        can_fuse = self.fast_store and self.splits == 1 and bn == 1 and n_out <= 65536
        self.sums = None if not sums else 'fused' if can_fuse else 'finish' if self.splits > 1 else 'stats'
        self.refused = self.sums == 'stats' and (out_f32 or n_out % 8 or n_out > 2048)
        self.finish_vec = (4 if n_out % 4 == 0 else 1) if self.splits > 1 else None
        self.store = ('split' if self.splits > 1 else 'swapped' if self.swap else 'wide' if self.wide else
                      'staged' if self.fast_store else 'fragment')
        self.kernel = (SWAP_VOX if self.swap else self.block_n, int(dgrad), self.wide or self.swap, self.swap)
        self.launches = 1 + int(self.splits > 1) + int(self.sums == 'stats')

    def kernel_name(self):
        bn, bmn, wide, swap = self.kernel
        return f'og_conv_igemm_kernel<{bn}, {bmn}, {str(wide).lower()}, {str(swap).lower()}>'

    def describe(self):
        return (f'{self.kernel_name()} {self.store}: box {self.box}, {self.m_tiles}x{self.n_tiles} tiles, '
                f'{self.num_kb} k-blocks, {self.splits} split(s), finish VEC {self.finish_vec}, vec_ok {self.vec_ok}, '
                f'sums {self.sums}, {self.launches} launch(es)')


# ------------------------------------------------------------------------------------------------------------------
# the case table
# ------------------------------------------------------------------------------------------------------------------
def causal(k):
    return (k[0] - 1, (k[1] - 1) // 2, (k[2] - 1) // 2)


def fc(cin, cout, k, N, ext, pad=None, c1=0, bias='0', res=False, f32=False, sums=False, ws='full', ld_extra=8,
       data='int', hi=3, res_hi=3, bias_hi=20, density=1.0, expect=None):
    """A forward case: x0 [N, *ext, cin] (+ x1 [N, *ext, c1]) -> [N, *ext, cout]; bias names the biases passed."""
    return dict(op='fwd', cin=cin, cout=cout, k=k, N=N, ext=ext, pad=pad or causal(k), c1=c1, bias=bias, res=res,
                f32=f32, sums=sums, ws=ws, ld_extra=ld_extra, data=data, hi=hi, res_hi=res_hi, bias_hi=bias_hi,
                density=density, expect=expect or {}, w_rows=cout, k_off=0)


def dc(cout, cin, k, N, ext, pad=None, w_rows=None, k_off=0, f32=False, ws='full', ld_extra=8, data='int', hi=3,
       density=1.0, expect=None):
    """A data-gradient case: dy [N, *ext, cout] -> dx [N, *ext, cin], weights [cout][ldw] with the segment at k_off."""
    return dict(op='dgrad', cin=cin, cout=cout, k=k, N=N, ext=ext, pad=pad or causal(k), c1=0, bias='', res=False,
                f32=f32, sums=False, ws=ws, ld_extra=ld_extra, data=data, hi=hi, res_hi=0, bias_hi=0,
                density=density, expect=expect or {}, w_rows=w_rows or cout, k_off=k_off)


K1, K3, K133, K311, K5 = ONE, (3, 3, 3), (1, 3, 3), (3, 1, 1), (5, 5, 5)


def kern(bn, bmn, wide=False, swap=False):
    return (bn, bmn, wide, swap)


# swapped tiles need >= 4 * 256 * SMs voxels per launch: 33 samples of 4 x 32 x 32 = 135168 >= 4 * 256 * 132
SWAP_N, SWAP_EXT = 33, (4, 32, 32)

CASES = {
    # ---- kernel instantiations and tiles
    'bn16_cout3_f32_frag': fc(128, 3, K3, 2, (3, 9, 13), f32=True, ws=0,
                              expect=dict(kernel=kern(16, 0), store='fragment', vec_ok=False, partial='wh')),
    'bn16_cout16_bf16_frag_res_bias1': fc(64, 16, K133, 3, (2, 5, 7), bias='1', res=True,
                                          expect=dict(kernel=kern(16, 0), store='fragment', vec_ok=True)),
    'bn32_cout18_f32_head_1x1': fc(512, 18, K1, 2, (2, 4, 4), pad=(0, 0, 0), f32=True,
                                   expect=dict(kernel=kern(32, 0), store='fragment', vec_ok=False, splits=1)),
    'bn64_staged_sums_sym_pad': fc(64, 64, K3, 2, (4, 8, 16), pad=(1, 1, 1), sums=True, hi=1, bias_hi=2, density=0.25,
                                   expect=dict(kernel=kern(64, 0), store='staged', sums='fused')),
    'bn64_cout48_frag_res': fc(64, 48, K3, 2, (3, 6, 10), res=True, bias='01',
                               expect=dict(kernel=kern(64, 0), store='fragment', vec_ok=True)),
    'bn128_staged_res_sums': fc(128, 128, K3, 2, (3, 10, 12), res=True, sums=True, hi=1, bias_hi=2, density=0.25,
                                expect=dict(kernel=kern(128, 0), store='staged', sums='fused', partial='wh')),
    'bn128_staged_res_big': fc(64, 128, K133, 2, (3, 10, 12), pad=(0, 1, 1), res=True, res_hi=3000, hi=6,
                               bias='01', expect=dict(kernel=kern(128, 0), store='staged')),
    'bn128_staged_shortcut_sums': fc(128, 128, K3, 2, (2, 6, 20), c1=64, bias='01', sums=True, hi=1, bias_hi=2,
                                     density=0.25, ws=0, expect=dict(kernel=kern(128, 0), store='staged',
                                                                     sums='fused')),
    'bn128_two_n_tiles_bias_none': fc(64, 192, K311, 2, (5, 6, 10), bias='', ws=0,
                                      expect=dict(kernel=kern(128, 0), store='staged', n_tiles=2)),
    'wide_sums': fc(64, 256, K3, 1, (4, 8, 16), pad=(1, 1, 1), sums=True, hi=1, bias_hi=2, density=0.125,
                    expect=dict(kernel=kern(256, 0, True), store='wide', sums='fused')),
    'wide_cout320_shortcut_res_sums': fc(64, 320, K133, 2, (2, 8, 8), pad=(0, 1, 1), c1=64, bias='01', res=True,
                                         sums=True, hi=1, bias_hi=2, res_hi=1, density=0.25,
                                         expect=dict(kernel=kern(256, 0, True), store='wide', n_tiles=2,
                                                     sums='fused')),
    'wide_big': fc(64, 256, K1, 2, (3, 3, 5), pad=(0, 0, 0), hi=8, res=True, res_hi=2000, bias='1',
                   expect=dict(kernel=kern(256, 0, True), store='wide', partial='wht')),
    'swapped_shortcut_sums': fc(64, 128, K133, SWAP_N, SWAP_EXT, pad=(0, 1, 1), c1=64, bias='01', sums=True, hi=1,
                                bias_hi=1, density=1 / 32, expect=dict(kernel=kern(256, 0, True, True),
                                                                       store='swapped', sums='fused')),
    'swapped_big_bias0': fc(64, 128, K1, SWAP_N, SWAP_EXT, pad=(0, 0, 0), hi=12, bias_hi=300,
                            expect=dict(kernel=kern(256, 0, True, True), store='swapped')),
    # ---- fragment stores: vec_ok true / false, fp32 / bf16, with and without a residual
    **{f'frag_cout{co}_{"f32" if f32 else "bf16"}{"_res" if r else ""}':
       fc(64, co, K3, 2, (3, 6, 9), res=r, f32=f32, res_hi=600 if r and not f32 else 3, bias='01' if r else '1',
          expect=dict(store='fragment', vec_ok=co == 96, kernel=kern(128 if co == 96 else 32, 0)))
       for co in (18, 96) for f32 in (False, True) for r in (False, True)},
    # ---- split-K finish pass
    'split_f32_vec4': fc(128, 64, K3, 2, (2, 4, 8), f32=True, expect=dict(split=True, finish_vec=4, splits=6)),
    'split_bf16_vec4_shortcut_sums_bias1': fc(128, 64, K3, 2, (3, 5, 7), c1=64, bias='1', sums=True, hi=1,
                                              bias_hi=2, expect=dict(split=True, finish_vec=4, sums='finish')),
    'split_bf16_vec4_big': fc(128, 128, K3, 1, (2, 4, 8), hi=6, bias='01', bias_hi=500,
                              expect=dict(split=True, finish_vec=4, store='split')),
    'split_bf16_vec1_sums': fc(128, 3, K3, 2, (2, 5, 6), sums=True, hi=2,
                               expect=dict(split=True, finish_vec=1, sums='finish')),
    'split_bf16_vec1_bias_none': fc(128, 18, K3, 1, (2, 3, 5), bias='', hi=4,
                                    expect=dict(split=True, finish_vec=1)),
    'split_f32_vec1_bias01': fc(128, 18, K3, 2, (2, 5, 6), f32=True, bias='01', expect=dict(split=True, finish_vec=1)),
    # ---- workspace sizes on a launch that splits 6 ways when it can; bn = 2 with N % bn != 0, so unsplit
    #      launches take their sums from og_gn_stats
    **{f'ws_{w}': fc(128, 64, K3, 3, (2, 4, 8), sums=True, hi=1, bias_hi=2, density=0.5, ws=w,
                     expect=dict(splits={0: 1, 'one': 1, 'two': 2, 'full': 6}[w],
                                 sums='finish' if w in ('two', 'full') else 'stats', bn_gt1=True))
       for w in (0, 'one', 'two', 'full')},
    # ---- og_gn_stats fallback
    'stats_bn4_N5': fc(64, 64, K3, 5, (2, 4, 4), pad=(1, 1, 1), sums=True, ws=0, hi=2,
                       expect=dict(sums='stats', bn_gt1=True, store='staged')),
    'stats_cout72': fc(64, 72, K133, 2, (3, 6, 10), pad=(0, 1, 1), sums=True, hi=1, bias_hi=2,
                       expect=dict(sums='stats', store='fragment', kernel=kern(128, 0))),
    # ---- geometry
    'k555_sym': fc(64, 64, K5, 1, (6, 7, 9), pad=(2, 2, 2), ws=0, hi=2, expect=dict(splits=1)),
    'k555_causal_sums': fc(64, 64, K5, 1, (5, 6, 7), sums=True, ws=0, hi=1, density=0.25, bias_hi=2),
    'k111_T1_H1_N1': fc(64, 64, K1, 1, (1, 1, 3), pad=(0, 0, 0), f32=True, expect=dict(bn_gt1=True)),
    'k311_pt0_partial_wht_sums': fc(64, 64, K311, 2, (5, 3, 9), pad=(0, 0, 0), sums=True, hi=1, bias_hi=3,
                                    expect=dict(partial='wht', sums='fused', store='staged')),
    'k311_causal_W1': fc(64, 64, K311, 3, (6, 7, 1), expect=dict(store='staged')),
    'k133_T1': fc(128, 64, K133, 2, (1, 9, 11), pad=(0, 1, 1), f32=True, bias='01'),
    # ---- data gradient
    'dgrad_bn64_wrows40_pitch': dc(64, 64, K3, 2, (3, 5, 7), pad=(1, 1, 1), w_rows=40, ld_extra=24, ws=0,
                                   expect=dict(kernel=kern(64, 1), store='staged')),
    'dgrad_bn128_k555_f32_split': dc(128, 128, K5, 1, (5, 6, 7), f32=True, hi=2,
                                     expect=dict(kernel=kern(128, 1), split=True, finish_vec=4)),
    'dgrad_bn128_k555_f32_unsplit': dc(128, 128, K5, 1, (5, 6, 7), f32=True, ws=0, hi=2,
                                       expect=dict(kernel=kern(128, 1), store='fragment', vec_ok=True)),
    'dgrad_cin192_two_n_tiles': dc(64, 192, K311, 2, (5, 6, 10), pad=(1, 0, 0), ws=0,
                                   expect=dict(kernel=kern(128, 1), n_tiles=2, store='staged')),
    'dgrad_k_off_shortcut': dc(128, 64, K1, 2, (4, 8, 8), pad=(0, 0, 0), k_off=27 * 128,
                               expect=dict(kernel=kern(64, 1))),
    'dgrad_k_off_wrows100_f32': dc(128, 128, K1, 2, (3, 5, 6), pad=(0, 0, 0), k_off=27 * 64, w_rows=100, f32=True,
                                   ld_extra=16, expect=dict(kernel=kern(128, 1))),
    'dgrad_split_bf16_N1': dc(256, 64, K3, 1, (2, 4, 4), expect=dict(split=True, finish_vec=4, bn_gt1=True)),
    'dgrad_wide': dc(128, 256, K3, 1, (4, 8, 16), ws=0, expect=dict(kernel=kern(256, 1, True), store='wide')),
    'dgrad_wide_wrows3_big': dc(64, 256, K311, 2, (3, 3, 5), w_rows=3, hi=40, ws=0,
                                expect=dict(kernel=kern(256, 1, True), partial='wht')),
    'dgrad_swapped': dc(64, 128, K133, SWAP_N, SWAP_EXT, pad=(0, 1, 1), w_rows=50,
                        expect=dict(kernel=kern(256, 1, True, True), store='swapped')),
    'dgrad_k311_pt0': dc(64, 64, K311, 2, (5, 3, 9), pad=(0, 0, 0), ws=0, expect=dict(partial='wht')),
    'dgrad_k333_causal_H1': dc(64, 64, K3, 2, (4, 1, 6), ws=0),
    # ---- bounded, real-valued operands
    'real_bn16_f32': fc(128, 3, K3, 2, (3, 9, 13), f32=True, ws=0, data='real'),
    'real_staged_res_sums': fc(128, 128, K3, 2, (3, 10, 12), res=True, sums=True, bias='01', data='real'),
    'real_frag96_bf16_res': fc(64, 96, K3, 2, (3, 6, 9), res=True, data='real'),
    'real_wide_shortcut_sums': fc(64, 256, K133, 2, (2, 8, 8), pad=(0, 1, 1), c1=64, sums=True, data='real'),
    'real_swapped': fc(64, 128, K1, SWAP_N, SWAP_EXT, pad=(0, 0, 0), bias='01', sums=True, data='real'),
    'real_split_bf16_sums': fc(128, 64, K3, 2, (3, 5, 7), c1=64, bias='1', sums=True, data='real',
                               expect=dict(split=True)),
    'real_split_f32_vec1': fc(128, 18, K3, 2, (2, 5, 6), f32=True, bias='01', data='real', expect=dict(split=True)),
    'real_stats_cout72': fc(64, 72, K133, 2, (3, 6, 10), pad=(0, 1, 1), sums=True, data='real'),
    'real_dgrad_k_off_wrows': dc(128, 64, K1, 2, (4, 8, 8), pad=(0, 0, 0), k_off=27 * 128, w_rows=72, data='real'),
    'real_dgrad_split_f32': dc(128, 128, K5, 1, (5, 6, 7), f32=True, data='real', expect=dict(split=True)),
    'real_dgrad_wide': dc(128, 256, K3, 1, (4, 8, 16), ws=0, data='real'),
    'real_dgrad_swapped': dc(64, 128, K1, SWAP_N, SWAP_EXT, pad=(0, 0, 0), data='real'),
}


def item_cases(sms):
    """The launches where the two consumers of a ping-pong CTA meet their edge cases (one 128-voxel sample per tile,
    27 k-blocks): one item per CTA, one item more than the grid, 3 per CTA + 1."""
    out = {}
    for name, rows in (('one_per_cta', sms // 2), ('grid_plus_one', sms + 1), ('three_per_cta_plus_one', 3 * sms + 1)):
        out[f'items_{name}_fwd'] = fc(64, 64, K3, rows, (1, 1, 128), sums=True, hi=1, bias_hi=2,
                                      expect=dict(items=rows, store='staged', sums='fused'))
        out[f'items_{name}_dgrad'] = dc(64, 64, K3, rows, (1, 1, 128), expect=dict(items=rows))
    return out


ITEM_NAMES = list(item_cases(132))


def case_of(name, sms):
    return CASES[name] if name in CASES else item_cases(sms)[name]


def ws_bytes_of(c, sms):
    ws = c['ws']
    if ws == 0:
        return 0
    if ws == 'full':
        return WS_FULL
    slab = c['N'] * math.prod(c['ext']) * c['cin' if c['op'] == 'dgrad' else 'cout'] * 4
    return slab * {'one': 1, 'two': 2}[ws]


def plan_of(c, sms):
    if c['op'] == 'fwd':
        return IgemmPlan(sms, False, c['cin'], c['k'], c['N'], c['ext'], c['cout'], c1=c['c1'], out_f32=c['f32'],
                         residual=c['res'], ws_bytes=ws_bytes_of(c, sms), sums=c['sums'])
    return IgemmPlan(sms, True, c['cout'], c['k'], c['N'], c['ext'], c['cin'], out_f32=c['f32'],
                     ws_bytes=ws_bytes_of(c, sms))


def assert_path(name, c, plan):
    for key, want in c['expect'].items():
        if key == 'split':
            got = plan.splits > 1
        elif key == 'bn_gt1':     # samples per tile > 1, and a last tile with fewer samples
            got = plan.box[3] > 1 and c['N'] % plan.box[3] != 0
        else:
            got = getattr(plan, key)
        assert got == want, f'{name}: {key} is {got}, the case is for {want}: {plan.describe()}'
    assert not plan.refused, name


# ------------------------------------------------------------------------------------------------------------------
# operands, calls and expectations
# ------------------------------------------------------------------------------------------------------------------
def make_inputs(c, seed, device=DEV):
    """Operands of a case, generated on the CPU (so that a CPU rehearsal sees the same data) and moved to `device`.
    Returns a dict; w is the [rows][ldw] weight matrix with NaN in the pitch columns and in the rows from w_rows on."""
    kind, hi, N, ext = c['data'], c['hi'], c['N'], c['ext']

    def op(shape, s, lo_hi=None, dtype=BF16, sparse=False, scale=1.0):
        h = hi if lo_hi is None else lo_hi
        t = operand(shape, s, kind, 'cpu', dtype, -h, h)
        if kind == 'real':
            t = t * scale
        if sparse and c['density'] < 1:
            g = torch.Generator().manual_seed(s + 1000)
            t = t * (torch.rand(shape, generator=g) < c['density']).to(dtype)
        return t.to(device)
    d = {}
    ntk = math.prod(c['k']) * c['cin']
    if c['op'] == 'fwd':
        d['x'] = op((N, *ext, c['cin']), seed, sparse=True)
        d['x1'] = op((N, *ext, c['c1']), seed + 1, sparse=True) if c['c1'] else None
        rows, cols = c['cout'], ntk + c['c1']
        ldw = cols + c['ld_extra']
        wreal = op((rows, cols), seed + 2)
        # real biases and residuals at 2^(0..20), the magnitudes of the products' sums, so that their mistakes show
        d['bias0'] = op((c['cout'],), seed + 3, c['bias_hi'], F32T, scale=2 ** 10) if '0' in c['bias'] else None
        d['bias1'] = op((c['cout'],), seed + 4, c['bias_hi'], F32T, scale=2 ** 10) if '1' in c['bias'] else None
        d['res'] = op((N, *ext, c['cout']), seed + 5, c['res_hi'], scale=2 ** 10) if c['res'] else None
        col0 = 0
    else:
        dy = op((N, *ext, c['cout']), seed, sparse=True)
        dy[..., c['w_rows']:] = 0              # the caller zero-pads dy's channels past the real weight rows
        d['dy'] = dy
        rows, col0 = c['w_rows'], c['k_off']
        cols = col0 + ntk
        ldw = cols + c['ld_extra']
        wreal = op((rows, cols), seed + 2)     # columns before k_off: the main taps of a packed row
    wg = Guarded((c['cout'], ldw), BF16, device=device)
    wg.t[:rows, :cols].copy_(wreal)
    d['wg'], d['ldw'], d['col0'] = wg, ldw, col0
    return d


def _call(name, *a):
    from open_genie_b200 import _lib
    _lib.call(name, *a, torch.cuda.current_stream().cuda_stream)


def _launches():
    from open_genie_b200 import _lib
    return _lib.launch_count()


def _p(t):
    return None if t is None else t.data_ptr()


def run(c, d, sms):
    """One call on guarded, NaN-filled outputs: (out, sums or None, launches)."""
    N, ext, k, pad = c['N'], c['ext'], c['k'], c['pad']
    n_out = c['cout'] if c['op'] == 'fwd' else c['cin']
    og = Guarded((N, *ext, n_out), F32T if c['f32'] else BF16)
    sg = Guarded((N, 2), F64T, init=torch.zeros(N, 2, dtype=F64T, device=DEV)) if c['sums'] else None
    wsb = ws_bytes_of(c, sms)
    wsg = Guarded((max(wsb // 4, 1),), F32T) if wsb else None
    ws = (wsg.ptr(), wsb) if wsb else (None, 0)
    n0 = _launches()
    if c['op'] == 'fwd':
        _call('og_conv3d_fwd', d['x'].data_ptr(), c['cin'], *k, *pad, _p(d['x1']), c['c1'], d['wg'].ptr(), d['ldw'],
              _p(d['bias0']), _p(d['bias1']), _p(d['res']), og.ptr(), int(c['f32']), N, *ext, c['cout'], *ws,
              None if sg is None else sg.ptr())
    else:
        _call('og_conv3d_dgrad', d['dy'].data_ptr(), c['cout'], c['w_rows'], d['wg'].ptr(), d['ldw'], c['k_off'], *k,
              *pad, og.ptr(), int(c['f32']), N, *ext, c['cin'], *ws)
    torch.cuda.synchronize()
    launches = _launches() - n0
    og.check_guard('out')
    if sg is not None:
        sg.check_guard('sums')
    if wsg is not None:
        wsg.check_guard('workspace')
    return og.t.clone(), None if sg is None else sg.t.clone(), launches


def reference(c, d):
    """(ref, mag): the float64 result and the same sum over |terms|."""
    k, pad, ext = c['k'], c['pad'], c['ext']
    wr = d['wg'].t[:c['w_rows']].double()
    ntk = math.prod(k) * c['cin']
    if c['op'] == 'fwd':
        w3 = wr[:, :ntk].reshape(c['cout'], -1, c['cin'])
        w1 = wr[:, ntk:ntk + c['c1']] if c['c1'] else None
        x, x1 = d['x'].double(), None if d['x1'] is None else d['x1'].double()
        bs = [b.double() for b in (d['bias0'], d['bias1']) if b is not None]
        res = None if d['res'] is None else d['res'].double()
        ref = fwd_ref(x, w3, k, ONE, pad, ext, x1=x1, w1=w1, biases=bs, residual=res)
        mag = fwd_ref(x.abs(), w3.abs(), k, ONE, pad, ext, x1=None if x1 is None else x1.abs(),
                      w1=None if w1 is None else w1.abs(), biases=[b.abs() for b in bs],
                      residual=None if res is None else res.abs())
        return ref, mag
    w3 = wr[:, c['k_off']:c['k_off'] + ntk].reshape(c['w_rows'], -1, c['cin'])
    dy = d['dy'].double()
    return (dgrad_ref(dy, w3, k, ONE, pad, ext, w_rows=c['w_rows']),
            dgrad_ref(dy.abs(), w3.abs(), k, ONE, pad, ext, w_rows=c['w_rows']))


def terms(c, plan):
    """Terms of an output's fp32 sum: the k-products, the split slabs, the biases and the residual."""
    return plan.num_kb * 64 + plan.splits + 3


def out_bound(c, plan, ref, mag):
    if c['data'] == 'int':
        assert mag.max() <= EXACT_LIMIT, 'case too large for the exact check'
        return (ref if c['f32'] else ref.to(BF16)), 0.0
    err = gam(terms(c, plan)) * SLACK * mag
    return ref, (err if c['f32'] else (1 + U) * err + U * ref.abs())


def sums_of(y):
    y = y.double().reshape(y.shape[0], -1)
    return torch.stack([y.sum(1), (y * y).sum(1)], 1), torch.stack([y.abs().sum(1), (y * y).sum(1)], 1)


def sums_bound(c, y):
    """(want, tol) for the GroupNorm sums of the kernel's own bf16 output y."""
    want, mag = sums_of(y)
    if c['data'] == 'int':
        assert mag.max() <= SUM_LIMIT, f'sums too large for the exact check: {mag.max().item()}'
        return want, 0.0
    return want, gam(y[0].numel() + 64) * SLACK * mag


def conv_case(name, c, sms):
    plan = plan_of(c, sms)
    assert_path(name, c, plan)
    print(f'{name} ({sms} SMs): {plan.describe()}')
    d = make_inputs(c, zlib.crc32(name.encode()))
    out, sums, launches = run(c, d, sms)
    assert launches == plan.launches, (name, launches, plan.describe())
    # the weights' pitch columns and the rows from w_rows on are NaN: had the kernel read one, the output would show it
    assert nan_bits(d['wg'].t[:, d['ldw'] - c['ld_extra']:]) and nan_bits(d['wg'].t[c['w_rows']:])
    ref, mag = reference(c, d)
    want, tol = out_bound(c, plan, ref, mag)
    check(f'{name} out', out, want, tol)
    if sums is not None:
        swant, stol = sums_bound(c, out)
        check(f'{name} sums', sums, swant, stol)
    out2, sums2, _ = run(c, d, sms)
    ity = Guarded.BITS[out.dtype][0]
    assert torch.equal(out.view(ity), out2.view(ity)), f'{name}: two runs differ'
    if sums is not None and c['data'] == 'int':
        assert torch.equal(sums, sums2), f'{name}: the sums of two runs differ'


@GPU
@pytest.mark.parametrize('name', list(CASES))
def test_conv_paths(name):
    conv_case(name, CASES[name], num_sms())


@GPU
@pytest.mark.parametrize('name', ITEM_NAMES)
def test_item_counts(name):
    sms = num_sms()
    conv_case(name, item_cases(sms)[name], sms)


# one case per kernel instantiation, finish-pass width and sums path: the profiler names what the mirror promised
PROFILED = ['bn16_cout3_f32_frag', 'bn32_cout18_f32_head_1x1', 'bn64_staged_sums_sym_pad', 'bn128_staged_res_sums',
            'wide_sums', 'swapped_shortcut_sums', 'split_bf16_vec4_shortcut_sums_bias1', 'split_bf16_vec1_sums',
            'stats_bn4_N5', 'dgrad_bn64_wrows40_pitch', 'dgrad_bn128_k555_f32_split', 'dgrad_wide', 'dgrad_swapped']


@GPU
def test_kernel_names():
    from torch.profiler import ProfilerActivity, profile
    sms = num_sms()
    for name in PROFILED:
        c = CASES[name]
        plan = plan_of(c, sms)
        d = make_inputs(c, zlib.crc32(name.encode()))
        run(c, d, sms)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(c, d, sms)
        names = [e.name for e in prof.events()]
        conv = {m.group(0) for m in (re.search(r'og_conv_igemm_kernel<[^>]*>', n) for n in names) if m}
        assert conv == {plan.kernel_name()}, (name, sorted(conv), plan.describe())
        fin = {m.group(1) for m in (re.search(r'og_splitk_finish_kernel<(\d)>', n) for n in names) if m}
        assert fin == ({str(plan.finish_vec)} if plan.splits > 1 else set()), (name, fin, plan.describe())
        stats = any('og_gn_stats' in n for n in names)
        assert stats == (plan.sums == 'stats'), (name, plan.describe())


@GPU
@pytest.mark.parametrize('op', ['fwd', 'dgrad'])
def test_wide_tile_keeps_the_bits_of_two_ping_pong_tiles(op):
    """DESIGN §3.1: the wide tile adds the k-blocks in the ping-pong order, so a 256-output layer on one 128 x 256 tile
    and as two 128-output launches on the ping-pong kernel give the same bits (real operands, where order matters)."""
    sms = num_sms()
    N, ext, k, pad = 1, (4, 8, 16), K3, (1, 1, 1)
    seed = zlib.crc32(f'wide_bits_{op}'.encode())
    if op == 'fwd':
        cin, ntk = 64, 27 * 64
        x = operand((N, *ext, cin), seed, 'real')
        w = operand((256, ntk), seed + 1, 'real')
        b = operand((256,), seed + 2, 'real', dtype=F32T)
        res = operand((N, *ext, 256), seed + 3, 'real')

        def call(rows, n_out):
            out = torch.empty((N, *ext, n_out), dtype=BF16, device=DEV)
            rs = res[..., rows].contiguous()
            _call('og_conv3d_fwd', x.data_ptr(), cin, *k, *pad, None, 0, w[rows].data_ptr(), ntk, b[rows].data_ptr(),
                  None, rs.data_ptr(), out.data_ptr(), 0, N, *ext, n_out, None, 0, None)
            return out
        plans = [IgemmPlan(sms, False, cin, k, N, ext, n, residual=True) for n in (256, 128)]
    else:
        cout = 128
        dy = operand((N, *ext, cout), seed, 'real')
        w = operand((cout, 27, 256), seed + 1, 'real')

        def call(cols, n_out):
            wc = w[:, :, cols].reshape(cout, -1).contiguous()
            out = torch.empty((N, *ext, n_out), dtype=BF16, device=DEV)
            _call('og_conv3d_dgrad', dy.data_ptr(), cout, cout, wc.data_ptr(), wc.shape[1], 0, *k, *pad, out.data_ptr(),
                  0, N, *ext, n_out, None, 0)
            return out
        plans = [IgemmPlan(sms, True, cout, k, N, ext, n) for n in (256, 128)]
    assert plans[0].store == 'wide' and plans[1].store == 'staged', [p.describe() for p in plans]
    whole = call(slice(0, 256), 256)
    lo, hi = call(slice(0, 128), 128), call(slice(128, 256), 128)
    torch.cuda.synchronize()
    assert torch.equal(whole.view(torch.int16), torch.cat([lo, hi], -1).view(torch.int16)), \
        'the wide tile and the ping-pong kernel give different bits'


# ------------------------------------------------------------------------------------------------------------------
# CPU: the case table and the mirror
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sms', [114, 132])
def test_cases_reach_their_paths(sms):
    for name in list(CASES) + list(item_cases(sms)):
        assert_path(name, case_of(name, sms), plan_of(case_of(name, sms), sms))


def _coverage(sms):
    """What the exact cases reach at `sms` SMs, as a set of path labels."""
    got = set()
    for name in list(CASES) + list(item_cases(sms)):
        c = case_of(name, sms)
        if c['data'] != 'int':
            continue
        p = plan_of(c, sms)
        dt = 'f32' if c['f32'] else 'bf16'
        got.add(('kernel', p.kernel))
        got.add(('store', p.store, c['op']))
        if p.splits > 1:
            got.add(('finish', p.finish_vec, dt, bool(c['sums'])))
        if p.store == 'staged':
            got.add(('staged', c['res'], c['sums']))
        if p.store == 'fragment':
            got.add(('fragment', p.vec_ok, dt, c['res']))
        if p.n_tiles > 1 and c['cout'] % p.block_n:
            got.add(('partial n tile', p.store))
        if c['op'] == 'fwd':
            got.add(('bias', c['bias'], p.store))
            got.add(('bias', c['bias']))
            if c['c1']:
                got.add(('second segment', p.store))
        got.add(('sums', p.sums, p.store))
        if p.sums == 'stats':
            got.add(('stats', 'bn>1, N % bn != 0' if p.box[3] > 1 and c['N'] % p.box[3] else
                     'cout % 64 != 0' if c['cout'] % 64 else 'other'))
        got.add(('ws', c['ws'], p.splits))
        got.add(('k', c['k'], c['op']))
        kt, pt = c['k'][0], c['pad'][0]
        if kt > 1:
            got.add(('pt', 'kt-1' if pt == kt - 1 else '(kt-1)/2' if pt == (kt - 1) // 2 else '0' if pt == 0 else pt))
        for a in p.partial:
            got.add(('partial box', a))
        if p.box[3] > 1 and c['N'] % p.box[3]:
            got.add(('bn > 1, N % bn != 0',))
        for a, e in zip('thw', c['ext']):
            if e == 1:
                got.add(('extent 1', a))
        if c['N'] == 1:
            got.add(('N = 1',))
        if c['op'] == 'dgrad':
            got.add(('dgrad', 'k_off' if c['k_off'] else 'k_off 0'))
            if c['w_rows'] < c['cout']:
                got.add(('dgrad', 'w_rows < cout'))
            if c['ld_extra']:
                got.add(('dgrad', 'pitch'))
            if c['f32']:
                got.add(('dgrad', 'f32'))
            if p.splits > 1:
                got.add(('dgrad', 'split'))
    return got


REQUIRED = (
    [('kernel', k) for k in (kern(16, 0), kern(32, 0), kern(64, 0), kern(128, 0), kern(64, 1), kern(128, 1),
                            kern(256, 0, True), kern(256, 1, True), kern(256, 0, True, True),
                            kern(256, 1, True, True))] +
    [('finish', v, dt, s) for v in (4, 1) for dt, s in (('bf16', True), ('bf16', False), ('f32', False))] +
    [('ws', 0, 1), ('ws', 'one', 1), ('ws', 'two', 2), ('ws', 'full', 6)] +
    [('staged', r, s) for r in (False, True) for s in (False, True)] +
    [('fragment', v, dt, r) for v in (False, True) for dt in ('f32', 'bf16') for r in (False, True)] +
    [('partial n tile', 'wide')] +
    [('bias', b) for b in ('', '0', '1', '01')] + [('bias', '1', 'split'), ('bias', '1', 'fragment')] +
    [('second segment', s) for s in ('staged', 'wide', 'swapped', 'split')] +
    [('sums', 'fused', s) for s in ('staged', 'wide', 'swapped')] + [('sums', 'finish', 'split')] +
    [('stats', 'bn>1, N % bn != 0'), ('stats', 'cout % 64 != 0')] +
    [('k', k, 'fwd') for k in (K1, K3, K133, K311, K5)] + [('k', k, 'dgrad') for k in (K1, K3, K133, K311, K5)] +
    [('pt', p) for p in ('kt-1', '(kt-1)/2', '0')] +
    [('partial box', a) for a in 'wht'] + [('bn > 1, N % bn != 0',)] + [('extent 1', a) for a in 'thw'] +
    [('N = 1',)] +
    [('dgrad', a) for a in ('k_off', 'w_rows < cout', 'pitch', 'f32', 'split')] +
    [('store', s, 'dgrad') for s in ('staged', 'fragment', 'wide', 'swapped', 'split')]
)


@pytest.mark.parametrize('sms', [114, 132])
def test_exact_cases_cover_every_path(sms):
    got = _coverage(sms)
    missing = [r for r in REQUIRED if r not in got]
    assert not missing, missing
    # the three item counts: one item per CTA, grid + 1, 3 * grid + 1
    items = {(c['op'], c['expect']['items']) for c in item_cases(sms).values()}
    assert items == {(op, n) for op in ('fwd', 'dgrad') for n in (sms // 2, sms + 1, 3 * sms + 1)}


@pytest.mark.parametrize('sms', [1, 8, 66, 114, 132])
def test_igemm_plan_invariants(sms):
    for dgrad in (False, True):
        for c0, n_out in ((64, 3), (64, 18), (128, 64), (64, 96), (64, 128), (256, 128), (128, 256), (512, 320),
                          (512, 512), (2048, 256), (64, 1024)):
            if dgrad and n_out % 64:
                continue
            for k in (K1, K3, K5):
                for N, ext in ((1, (1, 1, 3)), (2, (2, 4, 8)), (3, (3, 5, 7)), (8, (16, 32, 32)), (33, (4, 32, 32))):
                    for ws in (0, 1 << 20, WS_FULL):
                        for f32, res, sums in ((0, 0, 0), (1, 0, 0), (0, 1, 1), (0, 0, 1)):
                            if dgrad and (res or sums):
                                continue
                            p = IgemmPlan(sms, dgrad, c0, k, N, ext, n_out, out_f32=bool(f32), residual=bool(res),
                                          ws_bytes=ws, sums=bool(sums))
                            d = p.describe()
                            assert 1 <= p.splits <= 16 and p.splits <= max(1, p.num_kb // 8), d
                            assert p.splits == 1 or (p.splits * p.slab <= ws and not res and
                                                     p.splits * p.m_tiles * p.n_tiles <= sms * p.n_tiles), d
                            assert p.box[0] * p.box[1] * p.box[2] * p.box[3] == (SWAP_VOX if p.swap else TILE_M) or \
                                p.box[3] == 256, d
                            assert not p.swap or (p.splits == 1 and p.fast_store and p.n_tiles == 1), d
                            assert not p.wide or (p.splits == 1 and p.fast_store and not p.swap), d
                            assert p.n_tiles * p.block_n >= n_out and p.m_tiles >= 1, d
                            assert p.kernel[0] in (16, 32, 64, 128, 256) and (p.kernel[1] == 0 or p.kernel[0] >= 64), d
                            assert p.launches == 1 + (p.splits > 1) + (p.sums == 'stats'), d
                            assert p.sums != 'fused' or (p.box[3] == 1 and p.store in ('staged', 'wide', 'swapped'))
                            assert p.grid <= sms and p.items >= p.grid


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference against torch, at every stride-1 geometry of the table
# ------------------------------------------------------------------------------------------------------------------
def _geometries():
    return sorted({(c['k'], c['pad']) for c in CASES.values()})


@pytest.mark.parametrize('geom', _geometries(), ids=str)
def test_reference_matches_torch(geom):
    k, pad = geom
    for ext in ((1, 3, 2), (5, 7, 9), (4, 1, 6)):
        x = operand((2, *ext, 5), 11, 'real', 'cpu', F64T)
        w = operand((3, math.prod(k), 5), 12, 'real', 'cpu', F64T)
        dy = operand((2, *ext, 3), 13, 'real', 'cpu', F64T)
        for op, mine in (('fwd', fwd_ref(x, w, k, ONE, pad, ext)), ('dgrad', dgrad_ref(dy, w, k, ONE, pad, ext))):
            ref = torch_ref(op, x, w, dy, k, ONE, pad, ext)
            assert mine.shape == ref.shape, (op, ext, mine.shape, ref.shape)
            err = float((mine - ref).abs().max())
            assert err <= 1e-12 * float(ref.abs().max()), (op, geom, ext, err)


def test_reference_segments_biases_residual_and_w_rows():
    k, pad, ext = K3, causal(K3), (3, 4, 5)
    x = operand((2, *ext, 5), 21, 'real', 'cpu', F64T)
    x1 = operand((2, *ext, 4), 22, 'real', 'cpu', F64T)
    w = operand((6, 27, 5), 23, 'real', 'cpu', F64T)
    w1 = operand((6, 4), 24, 'real', 'cpu', F64T)
    b0, b1 = operand((6,), 25, 'real', 'cpu', F64T), operand((6,), 26, 'real', 'cpu', F64T)
    res = operand((2, *ext, 6), 27, 'real', 'cpu', F64T)
    dy = operand((2, *ext, 6), 28, 'real', 'cpu', F64T)
    full = fwd_ref(x, w, k, ONE, pad, ext, x1=x1, w1=w1, biases=[b0, b1], residual=res)
    want = torch_ref('fwd', x, w, dy, k, ONE, pad, ext) + torch.einsum('nthwc,oc->nthwo', x1, w1) + b0 + b1 + res
    assert float((full - want).abs().max()) <= 1e-12 * float(want.abs().max())
    dy4 = dy.clone()
    dy4[..., 4:] = 0
    got = dgrad_ref(dy, w, k, ONE, pad, ext, w_rows=4)
    want = torch_ref('dgrad', x, w, dy4, k, ONE, pad, ext)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


# ------------------------------------------------------------------------------------------------------------------
# CPU: the checks reject the mistakes they exist for
# ------------------------------------------------------------------------------------------------------------------
SENS_FWD = fc(128, 64, K3, 2, (3, 5, 7), c1=64, bias='01', res=True, sums=True)
SENS_DGRAD = dc(128, 64, K3, 2, (3, 5, 7), w_rows=100, k_off=64)


def _fwd_mistakes(c, d, plan):
    """The forward's output (float64, before rounding) as the kernel would produce it with each mistake, and a function
    that rounds like the kernel; the GroupNorm-sums mistake is separate."""
    k, pad, ext, cin, c1 = c['k'], c['pad'], c['ext'], c['cin'], c['c1']
    ntk = math.prod(k) * cin
    wr = d['wg'].t.double()
    w3 = wr[:, :ntk].reshape(c['cout'], -1, cin)
    x, x1 = d['x'].double(), d['x1'].double()
    b0, b1, res = d['bias0'].double(), d['bias1'].double(), d['res'].double()

    def y(w3_=w3, w1_=wr[:, ntk:ntk + c1], x_=x, bs=(b0, b1), r=res, mut=()):
        return fwd_ref(x_, w3_, k, ONE, pad, ext, mut, x1=x1, w1=w1_, biases=bs, residual=r)
    dropped = w3.clone()
    dropped[:, 13, :64] = 0                                # one k-block: channels 0-63 of the centre tap
    per_split = cdiv(plan.num_kb, 6)                       # as if the launch were split 6 ways
    first = w3.clone().reshape(c['cout'], -1)
    first[:, per_split * 64:] = 0                          # the k-blocks of split 0
    xh = d['x'].view(torch.float16).double()
    return {
        'a k-block dropped': y(w3_=dropped),
        'a split slab added twice': y() + fwd_ref(x, first.reshape(w3.shape), k, ONE, pad, ext),
        'causal padding applied symmetrically': y(mut=('causal_sym',)),
        'the shortcut segment read 8 columns early': y(w1_=wr[:, ntk - 8:ntk - 8 + c1]),
        'bias0 added twice': y(bs=(b0, b0, b1)),
        'bias1 added to the next column': y(bs=(b0, b1.roll(1))),
        'bf16 read as fp16': y(x_=torch.nan_to_num(xh, posinf=6e4, neginf=-6e4)),
    }


def _dgrad_mistakes(c, d):
    k, pad, ext, cin = c['k'], c['pad'], c['ext'], c['cin']
    ntk = math.prod(k) * cin
    wr = d['wg'].t[:c['w_rows']].double()
    dy = d['dy'].double()

    def g(off=c['k_off'], mut=(), dy_=dy):
        return dgrad_ref(dy_, wr[:, off:off + ntk].reshape(c['w_rows'], -1, cin), k, ONE, pad, ext, mut,
                         w_rows=c['w_rows'])
    return {
        'taps not mirrored': g(mut=('mirror',)),
        'causal padding applied symmetrically': g(mut=('causal_sym',)),
        'the segment read at k_off - 64': g(off=c['k_off'] - 64),
        'the segment read at k_off + 8': g(off=c['k_off'] + 8),
    }


def _rounded(c, v):
    return v if c['f32'] else v.to(BF16).double()


@pytest.mark.parametrize('data', ['real', 'int'])
def test_checks_reject_fwd_mistakes(data):
    c = dict(SENS_FWD, data=data, res_hi=600 if data == 'int' else 3)
    plan = plan_of(c, 132)
    d = make_inputs(c, 5, 'cpu')
    ref, mag = reference(c, d)
    want, tol = out_bound(c, plan, ref, mag)
    check('correct', ref.to(BF16), want, tol)
    for what, got in _fwd_mistakes(c, d, plan).items():
        rejects(lambda: check(what, _rounded(c, got), want, tol))
    # the residual added after the bf16 rounding of conv + bias
    conv = ref - d['res'].double()
    late = (conv.to(BF16).double() + d['res'].double()).to(BF16)
    rejects(lambda: check('residual added after rounding', late, want, tol))
    # overhang rows of a partial box counted in the GroupNorm sums: they hold bf16(bias0 + bias1). Integer data small
    # enough for the exact sums.
    if data == 'int':
        c = dict(c, hi=1, res_hi=1, bias_hi=2)
        d = make_inputs(c, 5, 'cpu')
        ref, _ = reference(c, d)
    y = ref.to(BF16)
    swant, stol = sums_bound(c, y)
    check('sums', sums_of(y)[0], swant, stol)
    bw, bh, bt, bn = plan.box
    T, H, W = c['ext']
    over = cdiv(T, bt) * bt * cdiv(H, bh) * bh * cdiv(W, bw) * bw - T * H * W
    assert over > 0
    b = (d['bias0'] + d['bias1']).to(BF16).double()
    wrong = sums_of(y)[0] + over * torch.stack([b.sum(), (b * b).sum()])
    rejects(lambda: check('overhang rows in the sums', wrong, swant, stol))


@pytest.mark.parametrize('data', ['real', 'int'])
def test_checks_reject_dgrad_mistakes(data):
    c = dict(SENS_DGRAD, data=data)
    plan = plan_of(c, 132)
    d = make_inputs(c, 6, 'cpu')
    ref, mag = reference(c, d)
    want, tol = out_bound(c, plan, ref, mag)
    check('correct', ref.to(BF16), want, tol)
    for what, got in _dgrad_mistakes(c, d).items():
        rejects(lambda: check(what, _rounded(c, got), want, tol))
    dyh = d['dy'].view(torch.float16).double()
    wr = d['wg'].t[:c['w_rows']].double()
    ntk = 27 * c['cin']
    fp16 = dgrad_ref(torch.nan_to_num(dyh, posinf=6e4, neginf=-6e4),
                     wr[:, 64:64 + ntk].reshape(c['w_rows'], -1, c['cin']), c['k'], ONE, c['pad'], c['ext'],
                     w_rows=c['w_rows'])
    rejects(lambda: check('bf16 read as fp16', _rounded(c, fp16), want, tol))


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument validation (host buffers, no CUDA call)
# ------------------------------------------------------------------------------------------------------------------
def test_fwd_dgrad_argument_validation_returns_status_codes():
    """Each call below breaks one condition and must return -1 with its message before any CUDA call: on a machine
    without a GPU a missing check ends in the tensor-map encoder's -3 instead."""
    from open_genie_b200 import _lib
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    p = (ctypes.addressof(buf) + 255) & ~255

    def bad(rc, text):
        assert rc == -1 and text in lib.og_last_error(), (rc, lib.og_last_error(), text)

    def dg(cout=64, w_rows=64, ldw=27 * 64, k_off=0, k=K3, pad=(2, 1, 1), cin=64, f32=0, ws=None, wsb=0):
        return lib.og_conv3d_dgrad(p, cout, w_rows, p, ldw, k_off, *k, *pad, p, f32, 1, 4, 8, 8, cin, ws, wsb, None)

    def fw(cout=64, f32=0, sums=p, ldw=27 * 64, ws=None, wsb=0):
        return lib.og_conv3d_fwd(p, 64, *K3, 2, 1, 1, None, 0, p, ldw, None, None, None, p, f32, 1, 4, 8, 8, cout, ws,
                                 wsb, sums, None)

    # data gradient: kernel extents and padding
    for k, pad in (((0, 3, 3), (0, 1, 1)), ((3, 0, 3), (2, 0, 1)), ((3, 3, -1), (2, 1, 0)), ((3, 3, 3), (3, 1, 1)),
                   ((3, 3, 3), (2, 3, 1)), ((3, 3, 3), (2, 1, 3)), ((3, 3, 3), (-1, 1, 1)), ((3, 3, 3), (2, -1, 1)),
                   ((1, 1, 1), (0, 0, 1))):
        bad(dg(k=k, pad=pad), b'conv3d_dgrad: bad kernel/padding')
    # k_off and the row pitch it needs
    bad(dg(k_off=-8, ldw=27 * 64 + 64), b'k_off=-8 must be >= 0')
    bad(dg(ldw=27 * 64 - 8), b'ldw=1720 must be >= k_off + kt*kh*kw*cin = 1728')
    bad(dg(k_off=64, ldw=27 * 64), b'ldw=1728 must be >= k_off + kt*kh*kw*cin = 1792')
    bad(dg(k=K1, pad=(0, 0, 0), k_off=27 * 128, ldw=27 * 128 + 56), b'must be >= k_off + kt*kh*kw*cin = 3520')
    # forward: GroupNorm sums need a bf16 output, and og_gn_stats's channel conditions when they are not fused
    bad(fw(f32=1), b'gn_sums needs a bf16 output')
    bad(fw(f32=1, ws=p, wsb=WS_FULL), b'gn_sums needs a bf16 output')
    bad(fw(cout=3), b'GroupNorm statistics of this launch')
    bad(fw(cout=2056, ldw=27 * 64), b'GroupNorm statistics of this launch')
    # the checks that already existed
    bad(dg(cout=72), b'cout=72 must be a multiple of 64')
    bad(dg(cin=96, ldw=27 * 96), b'cin=96 must be a multiple of 64')
    bad(dg(k_off=4, ldw=27 * 64 + 8), b'k_off/ldw must be multiples of 8')
    bad(dg(w_rows=65), b'w_rows=65 must be in (0, cout]')
    bad(fw(ldw=27 * 64 - 8), b'ldw=1720 must be >= 1728')
