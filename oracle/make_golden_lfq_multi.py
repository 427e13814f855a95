"""oracle/make_golden_lfq_multi.py — tests/golden/lfq_multi.pt by RUNNING THE REAL REFERENCE.   TEST INFRASTRUCTURE.

    OPEN_GENIE_REFERENCE=/path/to/open-genie python oracle/make_golden_lfq_multi.py

LookupFreeQuantization with num_codebook > 1 (genie/module/quantization.py:39-133), run as oracle/make_golden.py runs
its modules: unmodified reference, closed-form weights and inputs, CPU fp32. Every output, loss and gradient is
compared with oracle/lfq_multi_oracle.py (the literal restatement and the closed form; a mismatch aborts).
  * module cases: (D, C) in {(4, 2), (9, 2), (6, 3), (2, 4)}, each without projection, with a biased projection and
    with an unbiased one, on a 5-D input with transpose=True; train (loss, out, idxs, the gradients of
    loss + sum(out * g)) and eval (out, idxs);
  * the mini tokenizer (oracle.fixtures MINI_ENC / MINI_DEC, 6-channel latent) at (d_codebook, n_codebook) = (3, 2)
    (no projection) and (6, 2) (proj_inp / proj_out): tokenize quant and idxs, the training loss, every gradient's
    norm and samples, and the state_dict key list.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG                         # noqa: E402  (puts the reference and this repository on sys.path)
from make_golden import LookupFreeQuantization   # noqa: E402  (the reference's)
from make_golden import VideoTokenizer           # noqa: E402

from oracle import fixtures as fx                # noqa: E402
from oracle import genie_oracle as O             # noqa: E402
from oracle import lfq_multi_oracle as LM        # noqa: E402

MODULE_DC = ((4, 2), (9, 2), (6, 3), (2, 4))
# (tag, input_dim or None (passed as C * D: no projection; the reference's default is C * 2^D), use_bias)
PROJ = (('noproj', None, True), ('proj_bias', 16, True), ('proj_nobias', 16, False))
SHAPE = (2, None, 2, 3, 3)          # (b, input_dim, t, h, w), transpose=True: 36 tokens
X_SCALE = 0.01                      # 4 beta |x| ~ 4: codes from near 1 down to far below eps
TOKENIZER_DC = ((3, 2), (6, 2))
N_GRAD = 32                         # sampled elements of each tokenizer gradient


def sample(key, t, n):
    return t.detach().flatten()[O.det_indices(key, t.numel(), n)].clone()


def module_case(D, C, tag, input_dim, bias):
    name = f'd{D}c{C}_{tag}'
    idim = input_dim or C * D
    m = LookupFreeQuantization(D, num_codebook=C, input_dim=idim, use_bias=bias)
    sd = MG.load_det(m)
    shape = (SHAPE[0], idim) + SHAPE[2:]
    x = O.det_uniform(f'lfqm.x.{name}', shape, X_SCALE if input_dim is None else 1.0)
    gout = O.det_uniform(f'lfqm.g.{name}', shape, 1e-3)
    proj = lambda w: (sd[f'{w}.weight'], sd.get(f'{w}.bias')) if f'{w}.weight' in sd else None
    rec = {'D': D, 'C': C, 'input_dim': idim, 'bias': bias, 'shape': shape, 'keys': sorted(sd)}
    # train
    m.train()
    xr = x.clone().requires_grad_(True)
    (out, idxs), loss = m(xr, transpose=True)
    (loss + (out * gout).sum()).backward()
    grads = MG.grads_of(m)
    ref = {k: v.clone().requires_grad_(k in grads) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    pr = lambda w: (ref[f'{w}.weight'], ref.get(f'{w}.bias')) if f'{w}.weight' in ref else None
    (oout, oidx), oloss = LM.lfq(xo, D, C, True, transpose=True, proj_inp=pr('proj_inp'), proj_out=pr('proj_out'))
    (oloss + (oout * gout).sum()).backward()
    MG.close(oout, out, f'{name} train out'); MG.close(oidx, idxs, f'{name} idxs')
    MG.close(oloss, loss, f'{name} loss', rtol=1e-5, atol=1e-7)
    MG.close(xo.grad, xr.grad, f'{name} dx', rtol=1e-4, atol=1e-8)
    for k, g in grads.items():
        MG.close(ref[k].grad, g, f'{name} d {k}', rtol=1e-4, atol=1e-8)
    if input_dim is None:
        # the closed form of the kernels, in float64, on the quantiser's own input
        x2d = x.double().movedim(1, -1).reshape(-1, C * D)
        MG.close(LM.lfq_closed_form(x2d, D, C), loss.double(), f'{name} closed-form loss', rtol=1e-6, atol=1e-9)
    assert idxs.shape == shape[:1] + shape[2:] + (C,), idxs.shape
    rec.update(train={'out': out.detach(), 'idxs': idxs, 'loss': loss.detach(), 'dx': xr.grad.clone(),
                      'grads': {k: v.clone() for k, v in grads.items()}})
    # eval
    m.eval()
    (out, idxs), loss = m(x, transpose=True)
    assert loss is None
    (oout, oidx), _ = LM.lfq(x, D, C, False, transpose=True, proj_inp=proj('proj_inp'), proj_out=proj('proj_out'))
    MG.close(oout, out, f'{name} eval out'); MG.close(oidx, idxs, f'{name} eval idxs')
    rec['eval'] = {'out': out.detach(), 'idxs': idxs}
    return name, rec


def tokenizer_case(D, C):
    name = f'tok_d{D}c{C}'
    tok = VideoTokenizer(fx.bp(fx.MINI_ENC), fx.bp(fx.MINI_DEC), d_codebook=D, n_codebook=C, gan_loss_weight=0,
                         perc_loss_weight=0)
    tok.gan_crit = tok.perc_crit = MG.ZeroLoss()
    sd = MG.load_det(tok)
    keys = sorted(tok.state_dict())
    video = O.det_uniform('tokenizer.video', fx.MINI_VIDEO_SHAPE)
    quant, idxs = tok.tokenize(video)
    oq, oidx = LM.tokenizer_tokenize(sd, fx.MINI_ENC, video, D, C)
    MG.close(oq, quant, f'{name} tokenize quant'); MG.close(oidx, idxs, f'{name} tokenize idxs')
    tok.train()
    loss, (rec_loss, _, _, _, q_loss) = tok(video)
    loss.backward()
    oloss, (orec, oq_loss), _, _ = LM.tokenizer_forward(sd, fx.MINI_ENC, fx.MINI_DEC, video, D, C)
    MG.close(oloss, loss, f'{name} loss'); MG.close(orec, rec_loss, f'{name} rec loss')
    MG.close(oq_loss, q_loss, f'{name} quant loss')
    grads = MG.grads_of(tok)
    names = sorted(grads)
    enc = tok.encode(video).detach()
    return name, {'D': D, 'C': C, 'keys': keys, 'quant': quant, 'idxs': idxs, 'enc': enc, 'loss': loss.detach(),
                  'rec_loss': rec_loss.detach().clone(), 'quant_loss': q_loss.detach(), 'grad_names': names,
                  'grad_norm': {k: grads[k].norm().item() for k in names},
                  'grad': {k: sample(f'lfqm.{name}.{k}', grads[k], N_GRAD) for k in names}}


def main():
    out = {'module': {}, 'tokenizer': {}}
    for D, C in MODULE_DC:
        for tag, input_dim, bias in PROJ:
            name, rec = module_case(D, C, tag, input_dim, bias)
            out['module'][name] = rec
    for D, C in TOKENIZER_DC:
        name, rec = tokenizer_case(D, C)
        out['tokenizer'][name] = rec
    path = os.path.join(MG.OUT, 'lfq_multi.pt')
    torch.save(out, path)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
