"""Timing of BASELINE.json's parity-test configurations on one GPU (not bench.py lines): configs[0] tokenize()+decode(),
configs[2] LatentAction, configs[3] DynamicsModel, configs[4] Genie training steps — whole-step CUDA-event times plus a
per-kernel table (CUDA events around every C-ABI call; tensor-core kernels with their algorithmic TFLOP/s).

    python scripts/bench_configs.py [tokenize] [action] [dynamics] [genie]
"""
import collections, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import open_genie_b200 as og
from open_genie_b200 import _lib, ops


def kernel_table(steps):
    agg = collections.defaultdict(lambda: [0.0, 0])
    for name, _a, a, b in _lib.TIMING:
        agg[name][0] += a.elapsed_time(b) / steps
        agg[name][1] += 1
    return {k: {'ms': round(v[0], 3), 'launches': v[1] // steps} for k, v in sorted(agg.items(), key=lambda kv: -kv[1][0])}


def flop_table(steps):
    agg = collections.defaultdict(lambda: [0.0, 0.0])
    for kind, fl, a, b, _ in ops.PROFILE:
        agg[kind][0] += a.elapsed_time(b) / steps
        agg[kind][1] += fl / steps
    return {k: {'ms': round(v[0], 2), 'tflops': round(v[1] / max(v[0], 1e-9) * 1e-9, 1)} for k, v in agg.items()}


def run(name, model, step_fn, frames, steps=3, warm=2):
    params = [p for p in model.parameters() if p.requires_grad]
    opt = og.FusedAdamW(params)

    def step():
        loss = step_fn(); loss.backward(); opt.step(); opt.zero_grad(set_to_none=True); return loss
    for _ in range(warm):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    ops.PROFILE, _lib.TIMING = [], []
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    out = {'config': name, 'ms_per_step': round(ms, 2), 'frames_per_s': round(frames / ms * 1e3, 1), 'loss': float(loss),
           'params': sum(p.numel() for p in params), 'mem_gb': round(torch.cuda.max_memory_allocated() / 2**30, 1),
           'tensor_core_kernels': flop_table(steps), 'kernels_ms': kernel_table(steps)}
    ops.PROFILE, _lib.TIMING = None, None
    print(json.dumps(out), flush=True)


torch.manual_seed(0)
which = sys.argv[1:] or ['tokenize', 'action', 'dynamics', 'genie']
if 'tokenize' in which:
    # configs[0]: VideoTokenizer.tokenize() + decode() on (B,3,16,64,64) video, MAGVIT2 blueprints — inference path
    tok = og.VideoTokenizer(og.MAGVIT2_ENC_DESC, og.MAGVIT2_DEC_DESC, d_codebook=18, gan_loss_weight=0, perc_loss_weight=0).cuda()
    for B in (2, 8):
        v = torch.randn(B, 3, 16, 64, 64, device='cuda')

        def once():
            with torch.no_grad():
                q, idx = tok.tokenize(v)
                return tok.decode(q)
        for _ in range(3):
            once()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            once()
        e1.record(); torch.cuda.synchronize()
        ms_eager = e0.elapsed_time(e1) / 10
        side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            once()
        torch.cuda.current_stream().wait_stream(side); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            rec = once()
        g.replay(); torch.cuda.synchronize()
        e0.record()
        for _ in range(20):
            g.replay()
        e1.record(); torch.cuda.synchronize()
        ms_graph = e0.elapsed_time(e1) / 20
        _lib.TIMING = []
        once(); torch.cuda.synchronize()
        kt = kernel_table(1)
        _lib.TIMING = None
        print(json.dumps({'config': f'configs[0] VideoTokenizer.tokenize()+decode(), MAGVIT2, video ({B},3,16,64,64), bf16',
                          'ms_eager': round(ms_eager, 3), 'ms_graph_replay': round(ms_graph, 3),
                          'frames_per_s_graph': round(B * 16 / ms_graph * 1e3, 1), 'kernels_ms': kt}), flush=True)
        del g, rec
    del tok; torch.cuda.empty_cache()
if 'action' in which:
    B = int(os.environ.get('B_ACT', 16))
    la = og.LatentAction(og.LATENT_ACT_ENC, og.LATENT_ACT_DEC, d_codebook=8, n_embd=256, inp_shape=(64, 64)).cuda()
    v = torch.randn(B, 3, 16, 64, 64, device='cuda')
    run(f'configs[2] LatentAction fwd+bwd+AdamW, 8-action codebook, batch {B}x16x64x64', la, lambda: la(v)[1], B * 16)
    del la, v; torch.cuda.empty_cache()
if 'dynamics' in which:
    B, L = int(os.environ.get('B_DYN', 8)), int(os.environ.get('L_DYN', 8))
    dm = og.DynamicsModel((('space-time_attn', {'n_rep': L, 'n_head': 8, 'd_head': 64, 'transpose': False}),),
                          tok_vocab=1024, act_vocab=8, embed_dim=512).cuda()
    tok = torch.randint(0, 1024, (B, 16, 16, 16), device='cuda'); act = torch.randint(0, 8, (B, 16), device='cuda')
    mask = torch.rand(B, 16, 16, 16, device='cuda') < 0.75
    run(f'configs[3] DynamicsModel compute_loss step, L={L} ST blocks d=512 h=8, batch {B} of 16x16x16 tokens', dm,
        lambda: dm.compute_loss(tok, act, mask=mask), B * 16)
    del dm; torch.cuda.empty_cache()
if 'genie' in which:
    # configs[4]: frozen tokenizer WITHOUT temporal compression (REPR_TOK, d_codebook = 10 -> 16x16x16 tokens, vocab 1024):
    # token frames must equal action frames (genie/dynamics.py:55), see oracle/fixtures.py
    B = int(os.environ.get('B_GENIE', 16))
    tok = og.VideoTokenizer(og.REPR_TOK_ENC, og.REPR_TOK_DEC, d_codebook=10, gan_loss_weight=0, perc_loss_weight=0)
    gen = og.Genie(tok, dict(enc_desc=og.LATENT_ACT_ENC, dec_desc=og.LATENT_ACT_DEC, d_codebook=8, n_embd=256, inp_shape=(64, 64)),
                   dict(desc=(('space-time_attn', {'n_rep': 8, 'n_head': 8, 'd_head': 64, 'transpose': False}),),
                        tok_vocab=1024, act_vocab=256, embed_dim=512)).cuda()
    v = torch.randn(B, 3, 16, 64, 64, device='cuda')
    run(f'configs[4] Genie training_step (frozen REPR tokenizer d_codebook=10 + LatentAction + Dynamics L=8), per-GPU batch {B}',
        gen, lambda: gen.training_step(v, 0), B * 16)
