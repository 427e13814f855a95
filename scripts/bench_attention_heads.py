"""Times attention at head width 64 against head width 128 (default) or 16 (--narrow) on the same channel count C,
alternating the widths in one process (CUDA events, a window of launches per measurement, the median of --reps
alternations).

Flash attention (og_flash_attn_fwd / bwd, q = k = v with a residual, as the spatial attention calls it): ms per call
and algorithmic TFLOP/s with the FLOP counts of ops.py, 4 S^2 C per sequence forward and 10 S^2 C backward.
Temporal attention (og_temporal_attn_long_fwd / bwd, which d_head = 128 runs at every T): ms per call and the
bytes-over-time fraction of scripts/bench_temporal_attn.py. At T = 16 the d_head = 64 row is the kernel the model
runs there (the per-pixel kernels, og_temporal_attn_fwd / bwd); its bandwidth column uses the same byte count.

--narrow: 16 x 16 against 4 x 64 at C = 256. Flash rows add the exp-bound share: at d_head = 16 the softmax's exp2,
not the tensor cores, should bound the kernels. The forward evaluates one exp2 per score, the backward two (both
passes recompute P); the bound is that count at 16 exp2 results per clock per SM (the CUDA programming guide's
throughput table for compute capability 9.0) at clocks.max.sm, and the share is bound / measured time. Temporal
attention at d_head = 16 runs the tiled kernels at every T; at T = 16 the 4 x 64 row is the per-pixel kernels.

    python scripts/bench_attention_heads.py [--narrow] [--window 0.5] [--reps 3] [--json out.json]
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

from bench_temporal_attn import HBM, Problem, card, time_ms  # noqa: E402
from open_genie_b200 import _lib  # noqa: E402

DEV = 'cuda'


class Flash:
    def __init__(self, nseq, S, C, nh):
        self.nseq, self.S, self.C, self.nh = nseq, S, C, nh
        self.scale = nh * (C // nh) ** -0.5
        g = torch.Generator(device=DEV).manual_seed(1)
        rnd = lambda: (torch.randn((nseq, S, C), generator=g, device=DEV) * 0.5).to(torch.bfloat16)
        self.q, self.res, self.dout = rnd(), rnd(), rnd()
        self.out, self.out_res, self.dq, self.dk, self.dv = (torch.empty_like(self.q) for _ in range(5))
        self.lse = torch.empty((nseq, nh, S), device=DEV)
        self.delta = torch.empty_like(self.lse)
        self.s = torch.cuda.current_stream().cuda_stream

    def flops(self):
        return 4.0 * self.nseq * self.S ** 2 * self.C, 10.0 * self.nseq * self.S ** 2 * self.C

    def fwd(self):
        q = self.q.data_ptr()
        _lib.call('og_flash_attn_fwd', q, q, q, self.out.data_ptr(), self.res.data_ptr(), self.out_res.data_ptr(),
                  self.lse.data_ptr(), self.nseq, self.S, self.C, self.nh, self.scale, self.s)

    def bwd(self):
        q = self.q.data_ptr()
        _lib.call('og_flash_attn_bwd', q, q, q, self.out.data_ptr(), self.dout.data_ptr(), self.lse.data_ptr(),
                  self.delta.data_ptr(), self.dq.data_ptr(), self.dk.data_ptr(), self.dv.data_ptr(), self.nseq,
                  self.S, self.C, self.nh, self.scale, self.s)


def temporal(B, T, P, C, nh, bcast):
    pr = Problem(B, T, P, C, nh, bcast)
    pr.scale = nh * (C // nh) ** -0.5
    return pr


def alternate(fns, window, reps):
    """Median ms of each function, measured in turn `reps` times."""
    t = [[] for _ in fns]
    for _ in range(reps):
        for i, fn in enumerate(fns):
            t[i].append(time_ms(fn, window)[0])
    return [statistics.median(x) for x in t]


FLASH = [('dynamics-like', 128, 256, 512), ('latent-action full resolution', 32, 4096, 256)]
TEMPORAL = [(8, 16, 256, 512, 0), (8, 16, 256, 512, 1), (8, 64, 256, 512, 0), (8, 64, 256, 512, 1)]
FLASH_NARROW = [('latent-action 64x64 frames', 32, 4096, 256), ('16x16 frames', 128, 256, 256)]
TEMPORAL_NARROW = [(8, 16, 256, 256, 0), (8, 16, 256, 256, 1), (8, 64, 256, 256, 0), (8, 64, 256, 256, 1)]
EX2_PER_CLK_SM = 16


def max_sm_clock_mhz():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        return float(q.stdout.strip())
    except (OSError, subprocess.SubprocessError, ValueError):
        return None


def narrow(a):
    name, power = card()
    mhz = max_sm_clock_mhz()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f'card: {name}, power limit {power}, clocks.max.sm {mhz} MHz, {sms} SMs')
    ex2_rate = EX2_PER_CLK_SM * sms * mhz * 1e6 if mhz else None
    rows = []
    print(f'\nflash attention{"":26s} {"fwd ms":>8s} {"TFLOP/s":>8s} {"exp":>6s} {"bwd ms":>8s} {"TFLOP/s":>8s} '
          f'{"exp":>6s}')
    for label, nseq, S, C in FLASH_NARROW:
        probs = [Flash(nseq, S, C, C // d) for d in (16, 64)]
        f = alternate([p.fwd for p in probs], a.window, a.reps)
        for p in probs:
            p.fwd()
        b = alternate([p.bwd for p in probs], a.window, a.reps)
        for p, fm, bm in zip(probs, f, b):
            ff, bf = p.flops()
            n_ex2 = nseq * p.nh * S * S
            share = (lambda ms, n: n / ex2_rate / (ms * 1e-3) if ex2_rate else float('nan'))
            r = {'kind': 'flash', 'shape': label, 'nseq': nseq, 'S': S, 'C': C, 'n_head': p.nh, 'd_head': C // p.nh,
                 'fwd_ms': fm, 'fwd_tflops': ff / fm * 1e-9, 'fwd_exp_share': share(fm, n_ex2),
                 'bwd_ms': bm, 'bwd_tflops': bf / bm * 1e-9, 'bwd_exp_share': share(bm, 2 * n_ex2)}
            rows.append(r)
            tag = f'{label} {p.nh}x{C // p.nh}'
            print(f'{tag:41s} {fm:8.3f} {r["fwd_tflops"]:8.1f} {r["fwd_exp_share"]:6.2f} {bm:8.3f} '
                  f'{r["bwd_tflops"]:8.1f} {r["bwd_exp_share"]:6.2f}')
        del probs
        torch.cuda.empty_cache()
    print(f'\ntemporal attention, fraction of {HBM / 1e12:.2f} TB/s'
          f'{"":7s} {"fwd ms":>8s} {"fwd BW":>8s} {"bwd ms":>8s} {"bwd BW":>8s}')
    for B, T, P, C, bcast in TEMPORAL_NARROW:
        p16, p64 = temporal(B, T, P, C, C // 16, bcast), temporal(B, T, P, C, C // 64, bcast)
        short = T <= 32   # d_head 64 runs the per-pixel kernels there
        runs = [(p16, 'tiled', p16.long_fwd, p16.long_bwd),
                (p64, 'per-pixel', p64.lane_fwd, p64.lane_bwd) if short else (p64, 'tiled', p64.long_fwd, p64.long_bwd)]
        f = alternate([r[2] for r in runs], a.window, a.reps)
        p16.long_fwd()   # the tiled backward reads the forward's output and lse
        p64.long_fwd()
        b = alternate([r[3] for r in runs], a.window, a.reps)
        for (p, kern, _, _), fm, bm in zip(runs, f, b):
            fb, bb = p.bytes()
            d = C // p.nh
            r = {'kind': 'temporal', 'B': B, 'T': T, 'P': P, 'C': C, 'n_head': p.nh, 'd_head': d, 'kv_bcast': bcast,
                 'kernels': kern, 'fwd_ms': fm, 'fwd_bw_frac': fb / (fm * 1e-3) / HBM, 'bwd_ms': bm,
                 'bwd_bw_frac': bb / (bm * 1e-3) / HBM}
            rows.append(r)
            tag = f'T={T} {"bcast " if bcast else ""}{p.nh}x{d} ({kern})'
            print(f'{tag:41s} {fm:8.3f} {r["fwd_bw_frac"]:8.2f} {bm:8.3f} {r["bwd_bw_frac"]:8.2f}')
        del p16, p64, runs
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'clocks_max_sm_mhz': mhz, 'sms': sms, 'rows': rows}, f,
                      indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.5, help='seconds of launches per measurement')
    ap.add_argument('--reps', type=int, default=3, help='alternations of the two widths')
    ap.add_argument('--json', default=None, help='also write the results here')
    ap.add_argument('--narrow', action='store_true', help='16 x 16 against 4 x 64 heads instead of 64 against 128')
    a = ap.parse_args()
    if a.narrow:
        return narrow(a)
    name, power = card()
    print(f'card: {name}, power limit {power}')
    rows = []
    print(f'\nflash attention{"":26s} {"fwd ms":>8s} {"TFLOP/s":>8s} {"bwd ms":>8s} {"TFLOP/s":>8s}')
    for label, nseq, S, C in FLASH:
        probs = [Flash(nseq, S, C, C // d) for d in (64, 128)]
        f = alternate([p.fwd for p in probs], a.window, a.reps)
        for p in probs:   # the backward reads the forward's output and lse
            p.fwd()
        b = alternate([p.bwd for p in probs], a.window, a.reps)
        for p, fm, bm in zip(probs, f, b):
            ff, bf = p.flops()
            r = {'kind': 'flash', 'shape': label, 'nseq': nseq, 'S': S, 'C': C, 'n_head': p.nh, 'd_head': C // p.nh,
                 'fwd_ms': fm, 'fwd_tflops': ff / fm * 1e-9, 'bwd_ms': bm, 'bwd_tflops': bf / bm * 1e-9}
            rows.append(r)
            tag = f'{label} {p.nh}x{C // p.nh}'
            print(f'{tag:41s} {fm:8.3f} {r["fwd_tflops"]:8.1f} {bm:8.3f} {r["bwd_tflops"]:8.1f}')
        del probs
        torch.cuda.empty_cache()
    print(f'\ntemporal attention, fraction of {HBM / 1e12:.2f} TB/s'
          f'{"":7s} {"fwd ms":>8s} {"fwd BW":>8s} {"bwd ms":>8s} {"bwd BW":>8s}')
    for B, T, P, C, bcast in TEMPORAL:
        probs = [temporal(B, T, P, C, C // d, bcast) for d in (64, 128)]
        short = T <= 32   # d_head 64 runs the per-pixel kernels there
        fns_f = [probs[0].lane_fwd if short else probs[0].long_fwd, probs[1].long_fwd]
        fns_b = [probs[0].lane_bwd if short else probs[0].long_bwd, probs[1].long_bwd]
        f = alternate(fns_f, a.window, a.reps)
        probs[1].long_fwd()
        b = alternate(fns_b, a.window, a.reps)
        for p, fm, bm in zip(probs, f, b):
            fb, bb = p.bytes()
            d = C // p.nh
            kern = 'per-pixel' if short and d == 64 else 'tiled'
            r = {'kind': 'temporal', 'B': B, 'T': T, 'P': P, 'C': C, 'n_head': p.nh, 'd_head': d, 'kv_bcast': bcast,
                 'kernels': kern, 'fwd_ms': fm, 'fwd_bw_frac': fb / (fm * 1e-3) / HBM, 'bwd_ms': bm,
                 'bwd_bw_frac': bb / (bm * 1e-3) / HBM}
            rows.append(r)
            tag = f'T={T} {"bcast " if bcast else ""}{p.nh}x{d} ({kern})'
            print(f'{tag:41s} {fm:8.3f} {r["fwd_bw_frac"]:8.2f} {bm:8.3f} {r["bwd_bw_frac"]:8.2f}')
        del probs
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
