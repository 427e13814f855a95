"""Times one SpaceTimeAttention feed-forward block with a hidden layer (GroupNorm -> conv C->hid -> GELU -> conv hid->C,
+ x: ops.ffn_res), forward and backward, and the two GELU passes it runs (og_gelu_fwd / og_gelu_bwd) on their own.

CUDA events over a window of calls after warm-up; each figure is the median of --reps windows.
  conv TFLOP/s: algorithmic, forward 2 B T H W k^3 sum(Cin Cout) over the FFN's forward time, backward twice that over
                its backward time (the block's other passes, GroupNorm and GELU, count as time but not as FLOPs);
  GELU HBM    : bytes the pass must move (forward reads u, writes a: 4 B per element; backward reads da, u, writes
                du: 6 B) over its time, as a fraction of 3.35 TB/s;
  GELU share  : (GELU forward + backward) / (FFN forward + backward).
The backward time is (forward + backward) - forward, both measured.

    python scripts/bench_ffn.py [--window 0.5] [--reps 5] [--json out.json]
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

from bench_temporal_attn import HBM, card, time_ms  # noqa: E402
from open_genie_b200 import _lib, ops  # noqa: E402
from open_genie_b200.module.attention import _FfnNet  # noqa: E402

DEV = 'cuda'
# (name, B, T, H, W, C, hidden, k): the Dynamics transformer's width (embed_dim 512, 8 heads) at 16x16 tokens, and the
# LatentAction encoder's at 32x32
SHAPES = [
    ('dynamics_k3', 8, 16, 16, 16, 512, 2048, 3),
    ('dynamics_k1', 8, 16, 16, 16, 512, 2048, 1),
    ('latent_action_k3', 2, 16, 32, 32, 256, 1024, 3),
]


def measure(name, B, T, H, W, C, hid, k, window, reps):
    G = C // 64
    net = _FfnNet(C, C, (hid,), G, k, bias=False).to(DEV)
    gn = net.net[0]
    convs = [(c.weight, c.bias, c.packed(), c.geom) for c in (layer[0] for layer in net.net[1:])]
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn((B, T, H, W, C), generator=g, device=DEV).to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn((B, T, H, W, C), generator=g, device=DEV).to(torch.bfloat16)
    rows = B * T * H * W
    u = torch.randn((rows, hid), generator=g, device=DEV).to(torch.bfloat16)
    a, du = torch.empty_like(u), torch.empty_like(u)
    s = torch.cuda.current_stream().cuda_stream

    def fwd():
        return ops.ffn_res(x, gn.weight, gn.bias, convs, G, gn.eps)

    def fwd_bwd():
        x.grad = None
        net.zero_grad(set_to_none=True)
        fwd().backward(dy)

    runs = {'fwd': fwd, 'fwd_bwd': fwd_bwd,
            'gelu_fwd': lambda: _lib.call('og_gelu_fwd', u.data_ptr(), a.data_ptr(), rows, hid, s),
            'gelu_bwd': lambda: _lib.call('og_gelu_bwd', a.data_ptr(), u.data_ptr(), du.data_ptr(), rows, hid, s)}
    t = {n: [] for n in runs}
    for _ in range(reps):                      # alternate the measurements within each repetition
        for n, fn in runs.items():
            t[n].append(time_ms(fn, window)[0])
    ms = {n: statistics.median(v) for n, v in t.items()}
    ms['bwd'] = ms['fwd_bwd'] - ms['fwd']
    flops = 2.0 * rows * k ** 3 * (C * hid + hid * C)
    n = rows * hid
    res = {
        'shape': name, 'B': B, 'T': T, 'H': H, 'W': W, 'C': C, 'hidden': hid, 'k': k,
        'ffn_fwd_ms': ms['fwd'], 'ffn_bwd_ms': ms['bwd'],
        'conv_tflops_fwd': flops / ms['fwd'] * 1e-9, 'conv_tflops_bwd': 2 * flops / ms['bwd'] * 1e-9,
        'gelu_fwd_ms': ms['gelu_fwd'], 'gelu_bwd_ms': ms['gelu_bwd'],
        'gelu_fwd_hbm_frac': 4.0 * n / (ms['gelu_fwd'] * 1e-3) / HBM,
        'gelu_bwd_hbm_frac': 6.0 * n / (ms['gelu_bwd'] * 1e-3) / HBM,
        'gelu_share': (ms['gelu_fwd'] + ms['gelu_bwd']) / ms['fwd_bwd'],
    }
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--window', type=float, default=0.5, help='seconds of calls per measurement window')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--json', default=None, help='also write the results to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_ffn.py needs a CUDA device')
    name, power = card()
    print(f'card: {name}, power limit {power}')
    out = {'card': name, 'power_limit': power, 'results': []}
    for shape in SHAPES:
        r = measure(*shape, args.window, args.reps)
        out['results'].append(r)
        print(f"{r['shape']:18s} fwd {r['ffn_fwd_ms']:7.3f} ms ({r['conv_tflops_fwd']:5.0f} TFLOP/s)  "
              f"bwd {r['ffn_bwd_ms']:7.3f} ms ({r['conv_tflops_bwd']:5.0f} TFLOP/s)  "
              f"GELU fwd {r['gelu_fwd_ms']:.3f} ms ({r['gelu_fwd_hbm_frac']:.2f} of HBM)  "
              f"bwd {r['gelu_bwd_ms']:.3f} ms ({r['gelu_bwd_hbm_frac']:.2f})  share {100 * r['gelu_share']:.1f} %")
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
