"""Times the causal flash kernels against the non-causal ones, and the bidirectional tiled temporal kernels against the
causal temporal path the modules take, alternating the two in one process: CUDA events around a window of launches
per measurement, the median of --reps alternations.

Flash attention (og_flash_attn_causal_fwd / bwd against og_flash_attn_fwd / bwd, or og_flash_attn_dropout_fwd / bwd at
p = 0.1; q = k = v with a residual, as the spatial attention calls it) at d_head = 16, 64 and 128 on C = 256 channels
and S = 256, 1024 and 4096 tokens per frame (nseq * S = 32768 tokens), at p = 0 and 0.1. Temporal attention
(og_temporal_attn_bidir_fwd / bwd against the causal kernels ops._TimeAttnFn picks: the per-pixel
og_temporal_attn_fwd / bwd at d = 64, T = 16, og_temporal_attn_long_fwd / bwd otherwise) at T = 16 and 64 with B = 8,
256 pixels, C = 256 (16 heads of 16, 4 of 64, 2 of 128), without and with broadcast K / V, p = 0. Prints one row per
case (ms forward, ms backward, the ratio new / old) and writes them with the card's name and power limit to --json.

    python scripts/bench_attention_causal.py [--window 0.3] [--reps 3] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch  # noqa: E402

from bench_attention_dropout import Flash, Temporal  # noqa: E402
from bench_temporal_attn import card, time_ms  # noqa: E402
from open_genie_b200 import _lib, ops  # noqa: E402


class CausalFlash(Flash):
    """new: the causal kernels; old: the non-causal ones (with dropout at p > 0)."""

    def run(self, new, p, fwd):
        q = self.q.data_ptr()
        if fwd:
            args = (q, q, q, self.out.data_ptr(), self.res.data_ptr(), self.out_res.data_ptr(), self.lse.data_ptr(),
                    self.nseq, self.S, self.C, self.nh, self.scale)
        else:
            args = (q, q, q, self.out.data_ptr(), self.dout.data_ptr(), self.lse.data_ptr(), self.delta.data_ptr(),
                    self.dq.data_ptr(), self.dk.data_ptr(), self.dv.data_ptr(), self.nseq, self.S, self.C, self.nh,
                    self.scale)
        d = 'fwd' if fwd else 'bwd'
        if new:
            _lib.call(f'og_flash_attn_causal_{d}', *args, p, self.seed.data_ptr() if p > 0 else None, self.s)
        elif p > 0:
            (self.fwd if fwd else self.bwd)(p)
        else:
            _lib.call(f'og_flash_attn_{d}', *args, self.s)


class BidirTemporal(Temporal):
    """new: the bidirectional tiled kernels; old: the causal kernels ops._TimeAttnFn dispatches to."""

    def run(self, new, p, fwd):
        if fwd:
            args = (self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(), self.out.data_ptr(), self.res.data_ptr(),
                    self.out_res.data_ptr(), self.lse.data_ptr(), self.B, self.T, self.P, self.C, self.nh, self.scale,
                    self.bcast)
        else:
            dks = ((None, None, self.dkb.data_ptr(), self.dvb.data_ptr()) if self.bcast
                   else (self.dk.data_ptr(), self.dv.data_ptr(), None, None))
            args = (self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(), self.out.data_ptr(),
                    self.dout.data_ptr(), self.lse.data_ptr(), self.delta.data_ptr(), self.dq.data_ptr(), *dks, self.B,
                    self.T, self.P, self.C, self.nh, self.scale, self.bcast)
        d = 'fwd' if fwd else 'bwd'
        if new:
            _lib.call(f'og_temporal_attn_bidir_{d}', *args, p, None, self.s)
        elif ops._time_attn_tiled(self.T, self.C, self.nh):
            (self.fwd if fwd else self.bwd)(0.0)
        elif fwd:
            _lib.call('og_temporal_attn_fwd', self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                      self.res.data_ptr(), self.out_res.data_ptr(), self.B, self.T, self.P, self.C, self.nh,
                      self.scale, self.bcast, self.s)
        else:
            dks = ((None, None, self.dkb.data_ptr(), self.dvb.data_ptr()) if self.bcast
                   else (self.dk.data_ptr(), self.dv.data_ptr(), None, None))
            _lib.call('og_temporal_attn_bwd', self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                      self.dout.data_ptr(), self.dq.data_ptr(), *dks, self.B, self.T, self.P, self.C, self.nh,
                      self.scale, self.bcast, self.s)


def measure(pr, p, window, reps):
    """Median ms of fwd and bwd of the old and the new kernels, the two alternated `reps` times."""
    t = {k: [] for k in ('fwd_old', 'fwd_new', 'bwd_old', 'bwd_new')}
    pr.run(True, p, True)
    pr.run(False, p, True)
    for _ in range(reps):
        for new, tag in ((False, 'old'), (True, 'new')):
            t['fwd_' + tag].append(time_ms(lambda: pr.run(new, p, True), window)[0])
            t['bwd_' + tag].append(time_ms(lambda: pr.run(new, p, False), window)[0])
    return {k: statistics.median(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.3, help='seconds of launches per measurement')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    name, power = card()
    print(f'# {name}, power limit {power}; new (causal flash / bidirectional temporal) against old, median of '
          f'{args.reps} alternations')
    cases = [('flash', S, d, 0, p, lambda S=S, d=d: CausalFlash(S, d))
             for p in (0.0, 0.1) for d in (16, 64, 128) for S in (256, 1024, 4096)]
    cases += [('temporal', T, d, b, 0.0, lambda T=T, d=d, b=b: BidirTemporal(T, d, b))
              for d in (16, 64, 128) for T in (16, 64) for b in (0, 1)]
    print(f'{"kind":9s} {"S/T":>5s} {"d":>4s} {"bc":>3s} {"p":>4s} {"fwd old":>9s} {"fwd new":>9s} {"ratio":>6s} '
          f'{"bwd old":>9s} {"bwd new":>9s} {"ratio":>6s}')
    rows = []
    for kind, n, d, b, p, make in cases:
        pr = make()
        m = measure(pr, p, args.window, args.reps)
        row = dict(kind=kind, len=n, d_head=d, bcast=b, p=p, **m, fwd_ratio=m['fwd_new'] / m['fwd_old'],
                   bwd_ratio=m['bwd_new'] / m['bwd_old'])
        rows.append(row)
        print(f'{kind:9s} {n:5d} {d:4d} {b:3d} {p:4.1f} {m["fwd_old"]:9.3f} {m["fwd_new"]:9.3f} {row["fwd_ratio"]:6.2f} '
              f'{m["bwd_old"]:9.3f} {m["bwd_new"]:9.3f} {row["bwd_ratio"]:6.2f}', flush=True)
        del pr
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
