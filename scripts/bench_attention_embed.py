"""Times the LayerNorm-only row passes of attention without a rotary embedding (og_ln_rows_fwd / bwd, embed=False)
against the RoPE + LayerNorm passes they replace (og_rope_ln_fwd / bwd with the og_rope_table table, as ops.py calls
them), alternating the two in one process: CUDA events around a window of launches per measurement, the median of
--reps alternations.

Shapes: C = 256 channels. Spatial attention (positions = the S tokens of a frame) at S = 1024 and 4096 with 16 frames;
temporal attention (positions = the T frames of a pixel) at T = 16 and 64 with B = 8 clips of 256 pixels. The backward
passes take every gradient input (g0, g1, g2 and add), as the self-attention blocks call them. Each time is reported
against the HBM roofline: the bytes each pass must move (forward: read x, write y; backward: read x, g0, g1, g2, add,
write dx; bf16, the fp32 parameters and the cos / sin table neglected) over 3.35 TB/s, the H100 SXM data-sheet
bandwidth. Prints one row per case and writes them with the card's name, power limit and clocks to --json.

    python scripts/bench_attention_embed.py [--window 0.3] [--reps 5] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch  # noqa: E402

from bench_temporal_attn import card, time_ms  # noqa: E402
from open_genie_b200 import _lib  # noqa: E402
from oracle import genie_oracle as O  # noqa: E402

DEV = 'cuda'
HBM = 3.35e12     # bytes / s, H100 SXM data sheet


def clocks():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.max.sm,clocks.max.mem', '--format=csv,noheader', '-i',
                            '0'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


class Rows:
    """One row pass problem: rows of C channels at positions (row / pos_div) % pos_mod."""

    def __init__(self, kind, n, C=256):
        if kind == 'spatial':
            self.rows, self.pos_div, self.pos_mod, freq_kind = 16 * n, 1, n, '2d'
        else:
            self.rows, self.pos_div, self.pos_mod, freq_kind = 8 * n * 256, 256, n, '1d'
        self.C = C
        g = torch.Generator(device=DEV).manual_seed(1)
        rnd = lambda: torch.randn((self.rows, C), generator=g, device=DEV).to(torch.bfloat16)
        self.x, self.g0, self.g1, self.g2, self.add = (rnd() for _ in range(5))
        self.y, self.dx = torch.empty_like(self.x), torch.empty_like(self.x)
        self.gamma = 1 + 0.1 * torch.randn(C, generator=g, device=DEV)
        self.beta = 0.1 * torch.randn(C, generator=g, device=DEV)
        self.dgamma, self.dbeta = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        self.freq = O.rope_freq(C, freq_kind).to(DEV)
        self.tab = torch.empty((self.pos_mod, C // 2, 2), device=DEV)
        self.s = torch.cuda.current_stream().cuda_stream
        _lib.call('og_rope_table', self.freq.data_ptr(), self.pos_mod, C, self.tab.data_ptr(), self.s)

    def fwd(self, rope):
        if rope:
            _lib.call('og_rope_ln_fwd', self.x.data_ptr(), self.freq.data_ptr(), self.gamma.data_ptr(),
                      self.beta.data_ptr(), 1e-5, self.y.data_ptr(), self.rows, self.C, self.pos_div, self.pos_mod,
                      self.tab.data_ptr(), self.s)
        else:
            _lib.call('og_ln_rows_fwd', self.x.data_ptr(), self.gamma.data_ptr(), self.beta.data_ptr(), 1e-5,
                      self.y.data_ptr(), self.rows, self.C, self.s)

    def bwd(self, rope):
        grads = (self.g0.data_ptr(), self.g1.data_ptr(), self.g2.data_ptr(), self.add.data_ptr(), self.dx.data_ptr(),
                 self.dgamma.data_ptr(), self.dbeta.data_ptr(), self.rows, self.C)
        if rope:
            _lib.call('og_rope_ln_bwd', self.x.data_ptr(), self.freq.data_ptr(), self.gamma.data_ptr(), 1e-5, *grads,
                      self.pos_div, self.pos_mod, self.tab.data_ptr(), self.s)
        else:
            _lib.call('og_ln_rows_bwd', self.x.data_ptr(), self.gamma.data_ptr(), 1e-5, *grads, self.s)

    def bytes(self, which):
        return self.rows * self.C * 2 * (2 if which == 'fwd' else 6)


def measure(pr, window, reps):
    """Median ms of each pass with and without the rotation, the two alternated `reps` times."""
    t = {k: [] for k in ('fwd_rope', 'fwd_ln', 'bwd_rope', 'bwd_ln')}
    for _ in range(reps):
        for rope, tag in ((True, 'rope'), (False, 'ln')):
            t['fwd_' + tag].append(time_ms(lambda: pr.fwd(rope), window)[0])
            t['bwd_' + tag].append(time_ms(lambda: pr.bwd(rope), window)[0])
    return {k: statistics.median(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.3, help='seconds of launches per measurement')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    name, power = card()
    clk = clocks()
    print(f'# {name}, power limit {power}, max clocks (sm, mem) {clk}; median of {args.reps} alternations; '
          f'"roof" = HBM-roofline time / measured time')
    print(f'{"kind":8s} {"S/T":>5s} {"rows":>7s} {"fwd rope":>9s} {"fwd ln":>8s} {"roof":>5s} {"roof":>5s} '
          f'{"bwd rope":>9s} {"bwd ln":>8s} {"roof":>5s} {"roof":>5s}   (ms)')
    rows = []
    for kind, n in (('spatial', 1024), ('spatial', 4096), ('temporal', 16), ('temporal', 64)):
        pr = Rows(kind, n)
        m = measure(pr, args.window, args.reps)
        roof = {k: pr.bytes(k[:3]) / HBM * 1e3 / v for k, v in m.items()}
        rows.append(dict(kind=kind, len=n, rows=pr.rows, C=pr.C, **m, **{'roof_' + k: v for k, v in roof.items()}))
        print(f'{kind:8s} {n:5d} {pr.rows:7d} {m["fwd_rope"]:9.4f} {m["fwd_ln"]:8.4f} {roof["fwd_rope"]:5.2f} '
              f'{roof["fwd_ln"]:5.2f} {m["bwd_rope"]:9.4f} {m["bwd_ln"]:8.4f} {roof["bwd_rope"]:5.2f} '
              f'{roof["bwd_ln"]:5.2f}', flush=True)
        del pr
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'max_clocks_sm_mem': clk, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
