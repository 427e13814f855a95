"""Times the tiled temporal attention kernels (og_temporal_attn_long_fwd / bwd) at model shapes with CUDA events, and,
for information, against the per-pixel kernels (og_temporal_attn_fwd / bwd) at T = 32 on the same inputs.

Every shape is timed over enough launches for a window of at least one second after a warm-up. The bandwidth column
is algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s: every input row read once (q, k, v, the
residual; for the backward q, k, v, out, dout), every output written once (out, out_res; dq, dk, dv), plus the fp32
lse and delta (4 bytes per (row, head) each). Aliased inputs (k = v = q, as the product calls it) count once.

    python scripts/bench_temporal_attn.py [--window 1.0]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from open_genie_b200 import _lib  # noqa: E402

HBM = 3.35e12
DEV = 'cuda'


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power


def time_ms(fn, window):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    n = max(10, int(window * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n


class Problem:
    def __init__(self, B, T, P, C, nh, bcast):
        self.B, self.T, self.P, self.C, self.nh, self.bcast = B, T, P, C, nh, bcast
        self.scale = nh * 64 ** -0.5
        g = torch.Generator(device=DEV).manual_seed(1)
        rnd = lambda *s: torch.randn(*s, generator=g, device=DEV).to(torch.bfloat16)
        rows = (B, T, P, C)
        self.q = rnd(*rows)
        self.k, self.v = (rnd(B, T, C), rnd(B, T, C)) if bcast else (self.q, self.q)
        self.res, self.dout = rnd(*rows), rnd(*rows)
        self.out, self.out_res, self.dq = (torch.empty(rows, device=DEV, dtype=torch.bfloat16) for _ in range(3))
        self.dk, self.dv = (None, None) if bcast else (torch.empty_like(self.q), torch.empty_like(self.q))
        self.dkb = torch.zeros((B, T, C), device=DEV) if bcast else None
        self.dvb = torch.zeros((B, T, C), device=DEV) if bcast else None
        self.lse = torch.empty((B, nh, P, T), device=DEV)
        self.delta = torch.empty_like(self.lse)
        self.s = torch.cuda.current_stream().cuda_stream

    def bytes(self):
        row = self.B * self.T * self.P * self.C * 2
        kv = 2 * self.B * self.T * self.C * 2 if self.bcast else 0     # aliased k = v = q count with q
        kv_grad = 2 * self.B * self.T * self.C * 4 if self.bcast else 2 * row
        stat = self.B * self.T * self.P * self.nh * 4
        fwd = row + kv + row + 2 * row + stat                # q (k, v), residual; out, out_res; lse
        bwd = row + kv + 2 * row + stat + row + kv_grad + stat   # q (k, v), out, dout, lse; dq, dk, dv; delta
        return fwd, bwd

    def _p(self, t):
        return None if t is None else t.data_ptr()

    def long_fwd(self):
        _lib.call('og_temporal_attn_long_fwd', self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                  self.out.data_ptr(), self.res.data_ptr(), self.out_res.data_ptr(), self.lse.data_ptr(), self.B,
                  self.T, self.P, self.C, self.nh, self.scale, self.bcast, self.s)

    def long_bwd(self):
        _lib.call('og_temporal_attn_long_bwd', self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                  self.out.data_ptr(), self.dout.data_ptr(), self.lse.data_ptr(), self.delta.data_ptr(),
                  self.dq.data_ptr(), self._p(self.dk), self._p(self.dv), self._p(self.dkb), self._p(self.dvb),
                  self.B, self.T, self.P, self.C, self.nh, self.scale, self.bcast, self.s)

    def lane_fwd(self):
        _lib.call('og_temporal_attn_fwd', self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                  self.res.data_ptr(), self.out_res.data_ptr(), self.B, self.T, self.P, self.C, self.nh, self.scale,
                  self.bcast, self.s)

    def lane_bwd(self):
        _lib.call('og_temporal_attn_bwd', self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                  self.dout.data_ptr(), self.dq.data_ptr(), self._p(self.dk), self._p(self.dv), self._p(self.dkb),
                  self._p(self.dvb), self.B, self.T, self.P, self.C, self.nh, self.scale, self.bcast, self.s)


SHAPES = [
    # name, B, T, P, C, n_head, kv_bcast, backward
    ('dynamics T=64', 8, 64, 256, 512, 8, 0, True),
    ('dynamics T=256', 8, 256, 256, 512, 8, 0, True),
    ('latent-action T=64', 2, 64, 4096, 256, 4, 0, True),
    ('latent-action T=64 bcast', 2, 64, 4096, 256, 4, 1, True),
    ('roll-out T=1024', 1, 1024, 256, 512, 8, 0, False),
]
COMPARE_T32 = [
    ('dynamics T=32', 8, 32, 256, 512, 8, 0),
    ('latent-action T=32 bcast', 2, 32, 4096, 256, 4, 1),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=1.0, help='seconds of launches per timed shape')
    ap.add_argument('--json', default=None, help='also write the results here')
    a = ap.parse_args()
    name, power = card()
    print(f'card: {name}, power limit {power}; bandwidth fraction of {HBM / 1e12:.2f} TB/s')
    rows = []
    print(f'{"shape":28s} {"fwd ms":>9s} {"fwd BW":>7s} {"bwd ms":>9s} {"bwd BW":>7s}')
    for label, B, T, P, C, nh, bcast, bwd in SHAPES:
        pr = Problem(B, T, P, C, nh, bcast)
        fb, bb = pr.bytes()
        f_ms, _ = time_ms(pr.long_fwd, a.window)
        b_ms = None
        if bwd:
            b_ms, _ = time_ms(pr.long_bwd, a.window)
        r = {'shape': label, 'B': B, 'T': T, 'P': P, 'C': C, 'n_head': nh, 'kv_bcast': bcast, 'fwd_ms': f_ms,
             'fwd_bw_frac': fb / (f_ms * 1e-3) / HBM, 'bwd_ms': b_ms,
             'bwd_bw_frac': None if b_ms is None else bb / (b_ms * 1e-3) / HBM}
        rows.append(r)
        bs = '        -       -' if b_ms is None else f'{b_ms:9.3f} {r["bwd_bw_frac"]:7.2f}'
        print(f'{label:28s} {f_ms:9.3f} {r["fwd_bw_frac"]:7.2f} {bs}')
        del pr
        torch.cuda.empty_cache()
    print('\nT = 32, same inputs (information only): tiled (long) kernels vs per-pixel kernels')
    print(f'{"shape":28s} {"long fwd":>9s} {"lane fwd":>9s} {"long bwd":>9s} {"lane bwd":>9s}')
    for label, B, T, P, C, nh, bcast in COMPARE_T32:
        pr = Problem(B, T, P, C, nh, bcast)
        t = [time_ms(fn, a.window)[0] for fn in (pr.long_fwd, pr.lane_fwd, pr.long_bwd, pr.lane_bwd)]
        rows.append({'shape': label + ' (compare)', 'long_fwd_ms': t[0], 'lane_fwd_ms': t[1], 'long_bwd_ms': t[2],
                     'lane_bwd_ms': t[3]})
        print(f'{label:28s} {t[0]:9.3f} {t[1]:9.3f} {t[2]:9.3f} {t[3]:9.3f}')
        del pr
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as f:
            json.dump({'card': name, 'power_limit': power, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
