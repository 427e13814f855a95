"""Per-shape timing of the convolution forward / data-gradient GEMM (og_conv_igemm_kernel) through the C ABI.

Every forward and data-gradient shape class of the benchmark's VideoTokenizer step (B = 8, 16 x 64 x 64 clips) runs with
the epilogue the step uses there: bias pair, fused 1x1x1 shortcut segment, residual, GroupNorm sums, strided forward,
residue-class (strided) data gradient, split-K through the workspace, and the fp32 head and tail. Operands are seeded,
so the SHA-256 of every output identifies the result bit for bit across builds.

    python scripts/bench_conv_gemm.py --lib path/to/libopengenie_b200.so --out run.json
    python scripts/bench_conv_gemm.py --compare before.json after.json

--lib selects the shared library to load (default: the one built in the tree), so that two builds can be timed
alternately in one session and their outputs compared with --compare.
"""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, WS_BYTES = 8, 64 << 20

# (name, kind, arguments). fwd: cin, cout, k, (T, H, W), epilogue flags; sc = channels of the fused 1x1x1 shortcut.
SHAPES = [
    ('fwd 128->128 k3 @16x64x64 bias+gn', 'fwd', dict(cin=128, cout=128, k=3, grid=(16, 64, 64), bias=1, gn=True)),
    ('fwd 128->128 k3 @16x64x64 residual', 'fwd', dict(cin=128, cout=128, k=3, grid=(16, 64, 64), residual=True)),
    ('fwd 256->128 k3 @16x64x64 bias+gn', 'fwd', dict(cin=256, cout=128, k=3, grid=(16, 64, 64), bias=1, gn=True)),
    ('fwd 128->128 k3 +sc256 @16x64x64 bias2+gn', 'fwd',
     dict(cin=128, cout=128, k=3, grid=(16, 64, 64), sc=256, bias=2, gn=True)),
    ('fwd 256->256 k3 @16x32x32 bias+gn', 'fwd', dict(cin=256, cout=256, k=3, grid=(16, 32, 32), bias=1, gn=True)),
    ('fwd 256->1024 k3 @16x32x32 bias', 'fwd', dict(cin=256, cout=1024, k=3, grid=(16, 32, 32), bias=1)),
    ('fwd 256->256 k3 @8x16x16 bias+gn', 'fwd', dict(cin=256, cout=256, k=3, grid=(8, 16, 16), bias=1, gn=True)),
    ('fwd 512->512 k3 @4x8x8 bias+gn split-K', 'fwd', dict(cin=512, cout=512, k=3, grid=(4, 8, 8), bias=1, gn=True)),
    ('fwd 512->18 k1 @4x8x8 fp32 head', 'fwd', dict(cin=512, cout=18, k=1, grid=(4, 8, 8), bias=1, f32=True)),
    ('fwd 128->3 k3 @16x64x64 fp32 tail', 'fwd', dict(cin=128, cout=3, k=3, grid=(16, 64, 64), bias=1, f32=True)),
    ('strided fwd 128->128 k3 s(1,2,2) @16x64x64', 'sfwd', dict(cin=128, cout=128, k=3, s=(1, 2, 2), grid=(16, 64, 64))),
    ('dgrad 128<-128 k3 @16x64x64', 'dgrad', dict(cin=128, cout=128, k=3, grid=(16, 64, 64))),
    ('dgrad 256<-128 k3 @16x64x64', 'dgrad', dict(cin=256, cout=128, k=3, grid=(16, 64, 64))),
    ('dgrad 128<-3 k3 @16x64x64 (tail)', 'dgrad', dict(cin=128, cout=3, k=3, grid=(16, 64, 64))),
    ('dgrad 256<-256 k3 @16x32x32', 'dgrad', dict(cin=256, cout=256, k=3, grid=(16, 32, 32))),
    ('dgrad 256<-1024 k3 @16x32x32', 'dgrad', dict(cin=256, cout=1024, k=3, grid=(16, 32, 32))),
    ('dgrad 256<-256 k3 @8x16x16', 'dgrad', dict(cin=256, cout=256, k=3, grid=(8, 16, 16))),
    ('dgrad 512<-512 k3 @4x8x8 split-K', 'dgrad', dict(cin=512, cout=512, k=3, grid=(4, 8, 8))),
    ('strided dgrad 128<-128 k3 s(1,2,2) @16x64x64', 'sdgrad', dict(cin=128, cout=128, k=3, s=(1, 2, 2), grid=(16, 64, 64))),
    # the remaining classes with 256 or more output channels: decoder up-convolutions and channel changes
    ('fwd 128->256 k3 @16x32x32 bias+gn', 'fwd', dict(cin=128, cout=256, k=3, grid=(16, 32, 32), bias=1, gn=True)),
    ('fwd 256->256 k3 +sc128 @16x32x32 bias2+gn', 'fwd',
     dict(cin=256, cout=256, k=3, grid=(16, 32, 32), sc=128, bias=2, gn=True)),
    ('fwd 512->256 k3 @8x16x16 bias+gn', 'fwd', dict(cin=512, cout=256, k=3, grid=(8, 16, 16), bias=1, gn=True)),
    ('fwd 256->2048 k3 @8x16x16 bias', 'fwd', dict(cin=256, cout=2048, k=3, grid=(8, 16, 16), bias=1)),
    ('fwd 512->4096 k3 @4x8x8 bias', 'fwd', dict(cin=512, cout=4096, k=3, grid=(4, 8, 8), bias=1)),
    ('dgrad 256<-2048 k3 @8x16x16', 'dgrad', dict(cin=256, cout=2048, k=3, grid=(8, 16, 16))),
    ('dgrad 512<-256 k3 @8x16x16', 'dgrad', dict(cin=512, cout=256, k=3, grid=(8, 16, 16))),
]


def _rand(g, shape, dtype):
    import torch
    return ((torch.rand(shape, generator=g, device='cuda') * 2 - 1) * 0.5).to(dtype)


def _setup(name, kind, a):
    """Seeded operands and a closure that issues the call; returns (call, outputs to digest, gn sums or None, flop)."""
    import torch
    from open_genie_b200 import _lib
    bf16 = torch.bfloat16
    g = torch.Generator(device='cuda').manual_seed(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    cin, cout, k = a['cin'], a['cout'], a['k']
    T, H, W = a['grid']
    taps = k ** 3
    pt, ph = (k - 1, (k - 1) // 2)     # causal time padding, symmetric space padding
    ws = torch.empty(WS_BYTES, dtype=torch.uint8, device='cuda')
    s = torch.cuda.current_stream().cuda_stream
    if kind == 'fwd':
        sc = a.get('sc', 0)
        ldw = taps * cin + sc
        x = _rand(g, (B, T, H, W, cin), bf16)
        x1 = _rand(g, (B, T, H, W, sc), bf16) if sc else None
        w = _rand(g, (cout, ldw), bf16) * 0.1
        b0 = _rand(g, (cout,), torch.float32) if a.get('bias', 0) >= 1 else None
        b1 = _rand(g, (cout,), torch.float32) if a.get('bias', 0) >= 2 else None
        res = _rand(g, (B, T, H, W, cout), bf16) if a.get('residual') else None
        f32 = a.get('f32', False)
        out = torch.empty((B, T, H, W, cout), dtype=torch.float32 if f32 else bf16, device='cuda')
        sums = torch.zeros((B, 2), dtype=torch.float64, device='cuda') if a.get('gn') else None
        p = lambda t: None if t is None else t.data_ptr()   # noqa: E731

        def call():
            _lib.call('og_conv3d_fwd', x.data_ptr(), cin, k, k, k, pt, ph, ph, p(x1), sc, w.data_ptr(), ldw, p(b0), p(b1),
                      p(res), out.data_ptr(), int(f32), B, T, H, W, cout, ws.data_ptr(), WS_BYTES, p(sums), s)
        return call, out, sums, 2.0 * B * T * H * W * cout * ldw
    if kind == 'sfwd':
        st, sh, sw = a['s']
        pts = k - 1 + (1 - st)
        To, Ho, Wo = (T + pts - k) // st + 1, (H + 2 * ph - k) // sh + 1, (W + 2 * ph - k) // sw + 1
        x = _rand(g, (B, T, H, W, cin), bf16)
        w = _rand(g, (cout, taps * cin), bf16) * 0.1
        b0 = _rand(g, (cout,), torch.float32)
        out = torch.empty((B, To, Ho, Wo, cout), dtype=bf16, device='cuda')

        def call():
            _lib.call('og_conv3d_strided_fwd', x.data_ptr(), cin, k, k, k, st, sh, sw, pts, ph, ph, w.data_ptr(),
                      taps * cin, b0.data_ptr(), out.data_ptr(), 0, B, T, H, W, cout, s)
        return call, out, None, 2.0 * B * To * Ho * Wo * cout * taps * cin
    if kind == 'dgrad':
        cpad = (cout + 63) // 64 * 64     # dy channels padded to a multiple of 64; w has `cout` real rows
        dy = _rand(g, (B, T, H, W, cpad), bf16)
        w = _rand(g, (cout, taps * cin), bf16) * 0.1
        dx = torch.empty((B, T, H, W, cin), dtype=bf16, device='cuda')

        def call():
            _lib.call('og_conv3d_dgrad', dy.data_ptr(), cpad, cout, w.data_ptr(), taps * cin, 0, k, k, k, pt, ph, ph,
                      dx.data_ptr(), 0, B, T, H, W, cin, ws.data_ptr(), WS_BYTES, s)
        return call, dx, None, 2.0 * B * T * H * W * cin * taps * cout
    if kind == 'sdgrad':
        st, sh, sw = a['s']
        pts = k - 1 + (1 - st)
        To, Ho, Wo = (T + pts - k) // st + 1, (H + 2 * ph - k) // sh + 1, (W + 2 * ph - k) // sw + 1
        dy = _rand(g, (B, To, Ho, Wo, cout), bf16)
        w = _rand(g, (cout, taps * cin), bf16) * 0.1
        dx = torch.empty((B, T, H, W, cin), dtype=bf16, device='cuda')

        def call():
            _lib.call('og_conv3d_strided_dgrad', dy.data_ptr(), cout, cout, w.data_ptr(), taps * cin, k, k, k, st, sh, sw,
                      pts, ph, ph, dx.data_ptr(), B, T, H, W, cin, s)
        return call, dx, None, 2.0 * B * To * Ho * Wo * cout * taps * cin
    raise ValueError(kind)


def run(lib, iters, warmup):
    import torch
    from open_genie_b200 import _lib
    if lib:
        _lib.LIB_PATH = os.path.abspath(lib)
    _lib.load()
    rows = []
    for name, kind, a in SHAPES:
        call, out, sums, flop = _setup(name, kind, a)
        # the digested result: one call from zeroed GroupNorm sums
        call()
        torch.cuda.synchronize()
        digest = hashlib.sha256(out.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
        gn = sums.cpu().tolist() if sums is not None else None
        for _ in range(warmup):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        rows.append({'name': name, 'ms': ms, 'tflops': flop / (ms * 1e-3) * 1e-12, 'sha256': digest, 'gn_sums': gn})
        print(f'{name:48s} {ms:8.3f} ms {rows[-1]["tflops"]:7.1f} TFLOP/s  {digest[:16]}', flush=True)
        del call, out, sums
        torch.cuda.empty_cache()
    return rows


def compare(path_a, path_b):
    """Per-shape timing of two runs side by side, output digests, and the largest GroupNorm-sum difference."""
    a, b = (json.load(open(p)) for p in (path_a, path_b))
    ok = True
    print(f'{"shape":48s} {"A ms":>8s} {"B ms":>8s} {"B/A":>6s}  output  max rel. diff of GN sums')
    for ra, rb in zip(a['rows'], b['rows']):
        assert ra['name'] == rb['name']
        same = ra['sha256'] == rb['sha256']
        ok &= same
        gd = ''
        if ra['gn_sums'] is not None:
            d = max(abs(x - y) / max(abs(x), 1e-300) for pa, pb in zip(ra['gn_sums'], rb['gn_sums']) for x, y in zip(pa, pb))
            gd = f'{d:.2e}'
        print(f'{ra["name"]:48s} {ra["ms"]:8.3f} {rb["ms"]:8.3f} {rb["ms"] / ra["ms"]:6.3f}  '
              f'{"same" if same else "DIFFERS"}  {gd}')
    print('all outputs bit-identical' if ok else 'OUTPUTS DIFFER')
    return ok


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--lib', help='shared library to load (default: open_genie_b200/csrc/libopengenie_b200.so)')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', help='write the results as JSON')
    ap.add_argument('--compare', nargs=2, metavar=('A', 'B'), help='compare two --out files instead of running')
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_conv_gemm.py needs a CUDA device')
    rows = run(args.lib, args.iters, args.warmup)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'lib': args.lib, 'device': torch.cuda.get_device_name(), 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
