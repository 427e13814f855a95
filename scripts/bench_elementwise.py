"""Stand-alone timing of the HBM-bound GroupNorm passes at the largest tokenizer shape (CUDA events, L2 flushed
by cycling through more tensors than fit in L2)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from open_genie_b200 import _lib
N, V, C, G = 8, 16 * 64 * 64, int(os.environ.get('C', 128)), 1
dev = 'cuda'
K = 3  # rotating buffers: 3 x 134 MB x tensors > L2
xs = [torch.randn(N, V, C, device=dev).bfloat16() for _ in range(K)]
dys = [torch.randn(N, V, C, device=dev).bfloat16() for _ in range(K)]
adds = [torch.randn(N, V, C, device=dev).bfloat16() for _ in range(K)]
outs = [torch.empty(N, V, C, device=dev, dtype=torch.bfloat16) for _ in range(K)]
A = torch.randn(N, C, device=dev); Bc = torch.randn(N, C, device=dev)
gamma = torch.randn(C, device=dev); beta = torch.randn(C, device=dev)
mr = torch.rand(N, G, 2, device=dev) + 0.5
s = torch.cuda.current_stream().cuda_stream
def timeit(name, fn, bytes_):
    for i in range(3): fn(i % K)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    it = 12
    for i in range(it): fn(i % K)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / it
    print(f'{name:28s} {ms*1e3:8.1f} us  {bytes_/ms*1e-9:7.2f} TB/s')
T = N * V * C * 2
sums = torch.zeros(N, G, 2, dtype=torch.float64, device=dev)
S = torch.zeros(N, C, 2, device=dev)
dg = torch.zeros(C, device=dev); db = torch.zeros(C, device=dev); cs = torch.zeros(C, device=dev)
ws = torch.empty(64 << 20, dtype=torch.uint8, device=dev)   # partial sums of the reproducible reductions
timeit('gn_stats', lambda i: _lib.call('og_gn_stats', xs[i].data_ptr(), N, V, C, G, sums.data_ptr(), s), T)
timeit('gn_act_fwd', lambda i: _lib.call('og_gn_act_fwd', xs[i].data_ptr(), sums.data_ptr(), gamma.data_ptr(), beta.data_ptr(), None, None, 1e-5, G, 1, outs[i].data_ptr(), A.data_ptr(), Bc.data_ptr(), mr.data_ptr(), N, V, C, s), 2 * T)
A.normal_(); Bc.normal_(); mr.uniform_(0.5, 1.5)
timeit('bwd_reduce', lambda i: _lib.call('og_affine_act_bwd_reduce', dys[i].data_ptr(), xs[i].data_ptr(), A.data_ptr(), Bc.data_ptr(), 1, S.data_ptr(), N, V, C, ws.data_ptr(), ws.numel(), s), 2 * T)
timeit('gn_act_bwd', lambda i: _lib.call('og_gn_act_bwd', dys[i].data_ptr(), xs[i].data_ptr(), A.data_ptr(), Bc.data_ptr(), S.data_ptr(), mr.data_ptr(), gamma.data_ptr(), beta.data_ptr(), None, G, 1, None, outs[i].data_ptr(), dg.data_ptr(), db.data_ptr(), None, None, None, N, V, C, ws.data_ptr(), ws.numel(), s), 3 * T)
timeit('gn_act_bwd +add +colsum', lambda i: _lib.call('og_gn_act_bwd', dys[i].data_ptr(), xs[i].data_ptr(), A.data_ptr(), Bc.data_ptr(), S.data_ptr(), mr.data_ptr(), gamma.data_ptr(), beta.data_ptr(), None, G, 1, adds[i].data_ptr(), outs[i].data_ptr(), dg.data_ptr(), db.data_ptr(), None, None, cs.data_ptr(), N, V, C, ws.data_ptr(), ws.numel(), s), 4 * T)
timeit('colsum', lambda i: _lib.call('og_colsum', dys[i].data_ptr(), N * V, C, C, cs.data_ptr(), s), T)
y = torch.empty(N, V, C, device=dev, dtype=torch.bfloat16)
timeit('torch copy (ref)', lambda i: outs[i].copy_(xs[i]), 2 * T)
