"""Times the LFQ quantiser's training forward + backward (og_lfq_fwd + og_lfq_bwd at one codebook,
og_lfq_multi_fwd + og_lfq_multi_bwd at several) at the MAGVIT2 tokenizer's token count, B = 8 clips of 16 frames at
64 x 64 -> a 4 x 8 x 8 latent per clip = 2048 tokens, for (D, C) = (18, 1), (9, 2) and (6, 3): 2^18 code products per
token in the entropy term against C * 2^D. CUDA events around a window of launches per measurement; the cases are
alternated, and each row reports the median of --reps alternations. Prints one row per case and writes them with the
card's name and power limit to --json.

    python scripts/bench_lfq.py [--ntok 2048] [--window 0.3] [--reps 5] [--json out.json]
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
CASES = ((18, 1), (9, 2), (6, 3))
BETA, WC, WE, WD = 100.0, 0.25, 0.1, 1.0


class Lfq:
    def __init__(self, ntok, D, C):
        self.ntok, self.D, self.C = ntok, D, C
        g = torch.Generator(device=DEV).manual_seed(1)
        # unit-scale encoder outputs (the tokenizer's regime at beta = 100)
        self.x = torch.randn((ntok, C * D), generator=g, device=DEV)
        self.out = torch.empty_like(self.x)
        self.dx = torch.empty_like(self.x)
        self.idx = torch.empty((ntok, C), dtype=torch.int64, device=DEV)
        self.loss = torch.empty((1,), device=DEV)
        lib = _lib.load()
        nb = lib.og_lfq_workspace_bytes(ntok, D) if C == 1 else lib.og_lfq_multi_workspace_bytes(ntok, D, C)
        self.ws = torch.empty((nb,), dtype=torch.uint8, device=DEV)
        self.s = torch.cuda.current_stream().cuda_stream

    def step(self):
        x, n, D, C = self.x.data_ptr(), self.ntok, self.D, self.C
        if C == 1:
            _lib.call('og_lfq_fwd', x, D, n, D, BETA, 1, WC, WE, WD, self.out.data_ptr(), None, 0, self.idx.data_ptr(),
                      self.loss.data_ptr(), self.ws.data_ptr(), self.s)
            _lib.call('og_lfq_bwd', x, D, n, D, BETA, WC, WE, None, None, 0, self.dx.data_ptr(), None, D,
                      self.ws.data_ptr(), self.s)
        else:
            _lib.call('og_lfq_multi_fwd', x, C * D, n, D, C, BETA, 1, WC, WE, WD, self.out.data_ptr(), None, 0,
                      self.idx.data_ptr(), self.loss.data_ptr(), self.ws.data_ptr(), self.s)
            _lib.call('og_lfq_multi_bwd', x, C * D, n, D, C, BETA, WC, WE, None, None, 0, self.dx.data_ptr(), None,
                      C * D, self.ws.data_ptr(), self.s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ntok', type=int, default=2048)
    ap.add_argument('--window', type=float, default=0.3, help='seconds of launches per measurement')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_lfq.py needs a CUDA device'
    name, power = card()
    print(f'# {name}, power limit {power}; ntok = {args.ntok}')
    probs = {dc: Lfq(args.ntok, *dc) for dc in CASES}
    times = {dc: [] for dc in CASES}
    for _ in range(args.reps):
        for dc, p in probs.items():
            times[dc].append(time_ms(p.step, args.window)[0])
    rows = []
    for (D, C), ts in times.items():
        ms = statistics.median(ts)
        row = {'D': D, 'C': C, 'bits': C * D, 'code_products_per_token': C * 2 ** D, 'ntok': args.ntok,
               'ms_fwd_bwd': ms, 'spread_ms': [min(ts), max(ts)]}
        rows.append(row)
        print(f'D = {D:2d}  C = {C}  ({C * D} bits, {C * 2 ** D:6d} code products / token): '
              f'{ms:.4f} ms forward + backward  (min {min(ts):.4f}, max {max(ts):.4f})')
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
