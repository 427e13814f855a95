"""Times attention with dropout (p = 0.1) against the same call without it (p = 0, the entry points the modules call
at dropout 0), alternating the two in one process: CUDA events around a window of launches per measurement, the
median of --reps alternations.

Flash attention (og_flash_attn_[dropout_]fwd / bwd, q = k = v with a residual, as the spatial attention calls it) at
d_head = 16, 64 and 128 on C = 256 channels and S = 256, 1024 and 4096 tokens per frame (nseq * S = 32768 tokens), and
the tiled temporal kernels (og_temporal_attn_long_[dropout_]fwd / bwd) at T = 16 and 64 with B = 8, 256 pixels,
C = 256 (16 heads of 16, 4 of 64, 2 of 128), without and with broadcast K / V. Prints one row per case (ms forward,
ms backward, the ratio p = 0.1 / p = 0) and writes them with the card's name and power limit to --json.

    python scripts/bench_attention_dropout.py [--window 0.3] [--reps 3] [--json out.json]
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

from bench_temporal_attn import card, time_ms  # noqa: E402
from open_genie_b200 import _lib  # noqa: E402

DEV = 'cuda'
P_DROP = 0.1


class Flash:
    def __init__(self, S, d, C=256, tokens=32768):
        self.nseq, self.S, self.C, self.nh = tokens // S, S, C, C // d
        self.scale = self.nh * d ** -0.5
        g = torch.Generator(device=DEV).manual_seed(1)
        rnd = lambda: (torch.randn((self.nseq, S, C), generator=g, device=DEV) * 0.5).to(torch.bfloat16)
        self.q, self.res, self.dout = rnd(), rnd(), rnd()
        self.out, self.out_res, self.dq, self.dk, self.dv = (torch.empty_like(self.q) for _ in range(5))
        self.lse = torch.empty((self.nseq, self.nh, S), device=DEV)
        self.delta = torch.empty_like(self.lse)
        self.seed = torch.tensor([0x5EED], dtype=torch.int64, device=DEV)
        self.s = torch.cuda.current_stream().cuda_stream

    def fwd(self, p):
        q = self.q.data_ptr()
        args = (q, q, q, self.out.data_ptr(), self.res.data_ptr(), self.out_res.data_ptr(), self.lse.data_ptr(),
                self.nseq, self.S, self.C, self.nh, self.scale)
        if p > 0:
            _lib.call('og_flash_attn_dropout_fwd', *args, p, self.seed.data_ptr(), self.s)
        else:
            _lib.call('og_flash_attn_fwd', *args, self.s)

    def bwd(self, p):
        q = self.q.data_ptr()
        args = (q, q, q, self.out.data_ptr(), self.dout.data_ptr(), self.lse.data_ptr(), self.delta.data_ptr(),
                self.dq.data_ptr(), self.dk.data_ptr(), self.dv.data_ptr(), self.nseq, self.S, self.C, self.nh,
                self.scale)
        if p > 0:
            _lib.call('og_flash_attn_dropout_bwd', *args, p, self.seed.data_ptr(), self.s)
        else:
            _lib.call('og_flash_attn_bwd', *args, self.s)


class Temporal:
    def __init__(self, T, d, bcast, B=8, P=256, C=256):
        self.B, self.T, self.P, self.C, self.nh, self.bcast = B, T, P, C, C // d, bcast
        self.scale = self.nh * d ** -0.5
        g = torch.Generator(device=DEV).manual_seed(1)
        rnd = lambda *s: torch.randn(*s, generator=g, device=DEV).to(torch.bfloat16)
        rows = (B, T, P, C)
        self.q, self.res, self.dout = rnd(*rows), rnd(*rows), rnd(*rows)
        self.k, self.v = (rnd(B, T, C), rnd(B, T, C)) if bcast else (self.q, self.q)
        self.out, self.out_res, self.dq, self.dk, self.dv = (torch.empty_like(self.q) for _ in range(5))
        self.dkb, self.dvb = torch.zeros((B, T, C), device=DEV), torch.zeros((B, T, C), device=DEV)
        self.lse = torch.empty((B, self.nh, P, T), device=DEV)
        self.delta = torch.empty_like(self.lse)
        self.seed = torch.tensor([0x5EED], dtype=torch.int64, device=DEV)
        self.s = torch.cuda.current_stream().cuda_stream

    def fwd(self, p):
        args = (self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(), self.out.data_ptr(), self.res.data_ptr(),
                self.out_res.data_ptr(), self.lse.data_ptr(), self.B, self.T, self.P, self.C, self.nh, self.scale,
                self.bcast)
        if p > 0:
            _lib.call('og_temporal_attn_long_dropout_fwd', *args, p, self.seed.data_ptr(), self.s)
        else:
            _lib.call('og_temporal_attn_long_fwd', *args, self.s)

    def bwd(self, p):
        dks = ((None, None, self.dkb.data_ptr(), self.dvb.data_ptr()) if self.bcast
               else (self.dk.data_ptr(), self.dv.data_ptr(), None, None))
        args = (self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(), self.out.data_ptr(), self.dout.data_ptr(),
                self.lse.data_ptr(), self.delta.data_ptr(), self.dq.data_ptr(), *dks, self.B, self.T, self.P, self.C,
                self.nh, self.scale, self.bcast)
        if p > 0:
            _lib.call('og_temporal_attn_long_dropout_bwd', *args, p, self.seed.data_ptr(), self.s)
        else:
            _lib.call('og_temporal_attn_long_bwd', *args, self.s)


def measure(pr, window, reps):
    """Median ms of fwd and bwd at p = 0 and p = P_DROP, the two alternated `reps` times."""
    t = {k: [] for k in ('fwd0', 'fwdp', 'bwd0', 'bwdp')}
    pr.fwd(0.0)
    for _ in range(reps):
        for p, tag in ((0.0, '0'), (P_DROP, 'p')):
            t['fwd' + tag].append(time_ms(lambda: pr.fwd(p), window)[0])
            t['bwd' + tag].append(time_ms(lambda: pr.bwd(p), window)[0])
    return {k: statistics.median(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.3, help='seconds of launches per measurement')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    name, power = card()
    print(f'# {name}, power limit {power}; p = {P_DROP} against p = 0, median of {args.reps} alternations')
    rows = []
    cases = [('flash', S, d, 0, lambda S=S, d=d: Flash(S, d)) for d in (16, 64, 128) for S in (256, 1024, 4096)]
    cases += [('temporal', T, d, b, lambda T=T, d=d, b=b: Temporal(T, d, b)) for d in (16, 64, 128) for T in (16, 64)
              for b in (0, 1)]
    print(f'{"kind":9s} {"S/T":>5s} {"d":>4s} {"bc":>3s} {"fwd p=0":>9s} {"fwd p":>9s} {"ratio":>6s} '
          f'{"bwd p=0":>9s} {"bwd p":>9s} {"ratio":>6s}')
    for kind, n, d, b, make in cases:
        pr = make()
        m = measure(pr, args.window, args.reps)
        row = dict(kind=kind, len=n, d_head=d, bcast=b, **m, fwd_ratio=m['fwdp'] / m['fwd0'],
                   bwd_ratio=m['bwdp'] / m['bwd0'])
        rows.append(row)
        print(f'{kind:9s} {n:5d} {d:4d} {b:3d} {m["fwd0"]:9.3f} {m["fwdp"]:9.3f} {row["fwd_ratio"]:6.2f} '
              f'{m["bwd0"]:9.3f} {m["bwdp"]:9.3f} {row["bwd_ratio"]:6.2f}', flush=True)
        del pr
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'p': P_DROP, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
