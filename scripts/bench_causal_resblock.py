"""Times grouped blur pooling (og_blurpool3d_grouped) and causal against non-causal video residual blocks.

  blur    : forward and backward at B = 8, 128 channels, 16 x 64 x 64, k = 3, strides (1,2,2) and (2,2,2), groups 1, 2
            and 8 through og_blurpool3d_grouped, and groups = 1 through og_blurpool3d. HBM fraction: the bytes the
            pass must move (x read once, y written once; backward dy read once, dx written once, all bf16) over its
            time, as a fraction of 3.35 TB/s. The fp32 group sums it also writes and reads are not counted.
  block   : VideoResidualBlock(128, 128) forward + backward on (8, 128, 16, 64, 64), use_causal True against False
            (both take the fused single-node path). The convolutions do the same MACs; only the time padding differs.
CUDA events over a window of calls after warm-up; each figure is the median of --reps windows, and the variants are
alternated within each repetition.

    python scripts/bench_causal_resblock.py [--window 0.5] [--reps 5] [--json out.json]
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

from bench_temporal_attn import HBM, card, time_ms  # noqa: E402
from open_genie_b200 import _lib  # noqa: E402

DEV = 'cuda'
B, C, T, H, W, K = 8, 128, 16, 64, 64, 3


def clocks():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.max.sm,clocks.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def bench_blur(window, reps):
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn((B, T, H, W, C), generator=g, device=DEV).to(torch.bfloat16)
    s = torch.cuda.current_stream().cuda_stream
    rows = []
    for stride in ((1, 2, 2), (2, 2, 2)):
        st, sh, sw = stride
        To, Ho, Wo = (T - 1) // st + 1, (H - 1) // sh + 1, (W - 1) // sw + 1
        y = torch.empty((B, To, Ho, Wo, C), dtype=torch.bfloat16, device=DEV)
        dy = torch.randn((B, To, Ho, Wo, C), generator=g, device=DEV).to(torch.bfloat16)
        dx = torch.empty_like(x)
        scratch = torch.empty(B * T * H * W * 8, dtype=torch.float32, device=DEV)
        nbytes = 2 * (x.numel() + y.numel())
        runs = {}
        for G in (1, 2, 8):
            runs[f'grouped_G{G}_fwd'] = lambda G=G: _lib.call(
                'og_blurpool3d_grouped', x.data_ptr(), y.data_ptr(), scratch.data_ptr(), 0, B, T, H, W, C, C, G, K,
                st, sh, sw, s)
            runs[f'grouped_G{G}_bwd'] = lambda G=G: _lib.call(
                'og_blurpool3d_grouped', dy.data_ptr(), dx.data_ptr(), scratch.data_ptr(), 1, B, T, H, W, C, C, G, K,
                st, sh, sw, s)
        runs['og_blurpool3d_fwd'] = lambda: _lib.call('og_blurpool3d', x.data_ptr(), y.data_ptr(), scratch.data_ptr(),
                                                      0, B, T, H, W, C, C, K, st, sh, sw, s)
        runs['og_blurpool3d_bwd'] = lambda: _lib.call('og_blurpool3d', dy.data_ptr(), dx.data_ptr(), scratch.data_ptr(),
                                                      1, B, T, H, W, C, C, K, st, sh, sw, s)
        t = {n: [] for n in runs}
        for _ in range(reps):
            for n, fn in runs.items():
                t[n].append(time_ms(fn, window)[0])
        for n, v in t.items():
            ms = statistics.median(v)
            rows.append({'stride': stride, 'pass': n, 'ms': ms, 'hbm_frac': nbytes / (ms * 1e-3) / HBM,
                         'spread_ms': (min(v), max(v))})
    return rows


def bench_block(window, reps):
    from open_genie_b200.module.video import VideoResidualBlock
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn((B, C, T, H, W), generator=g, device=DEV).requires_grad_(True)
    blocks = {c: VideoResidualBlock(C, C, use_causal=c).to(DEV) for c in (False, True)}
    dy = None
    runs = {}
    for causal, m in blocks.items():
        def step(m=m):
            nonlocal dy
            x.grad = None
            m.zero_grad(set_to_none=True)
            y = m(x)
            if dy is None:
                dy = torch.randn_like(y)          # same (channels-last) strides as y
            y.backward(dy)
        runs['causal' if causal else 'plain'] = step
    t = {n: [] for n in runs}
    for _ in range(reps):
        for n, fn in runs.items():
            t[n].append(time_ms(fn, window)[0])
    return [{'block': n, 'fwd_bwd_ms': statistics.median(v), 'spread_ms': (min(v), max(v))} for n, v in t.items()]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--window', type=float, default=0.5, help='seconds of calls per measurement window')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', default=None, help='also write the results to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_causal_resblock.py needs a CUDA device')
    name, power = card()
    clk = clocks()
    print(f'card: {name}, power limit {power}, clocks.max.sm / clocks.sm {clk}')
    out = {'card': name, 'power_limit': power, 'clocks': clk, 'blur': bench_blur(args.window, args.reps),
           'block': bench_block(args.window, args.reps)}
    for r in out['blur']:
        print(f"blur stride {r['stride']}  {r['pass']:20s} {r['ms']:7.3f} ms  {r['hbm_frac']:.2f} of HBM  "
              f"(spread {r['spread_ms'][0]:.3f}-{r['spread_ms'][1]:.3f})")
    for r in out['block']:
        print(f"block 128->128 {r['block']:6s} fwd+bwd {r['fwd_bwd_ms']:7.3f} ms  "
              f"(spread {r['spread_ms'][0]:.3f}-{r['spread_ms'][1]:.3f})")
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
