"""oracle/lfq_multi_oracle.py — LookupFreeQuantization with num_codebook > 1, restated in plain torch.   TEST INFRASTRUCTURE.

Extends oracle.genie_oracle.lfq (num_codebook == 1) to any number of codebooks C (genie/module/quantization.py:39-133):
  * lfq: the literal forward. The C*D inputs of a token are split into C slices of D ('b n (c d) -> b n c d', line
    91), each slice gets its own MSB-first index (line 98), and the entropy loss runs over the reference's codebook of
    C * 2^D rows, row j the sign code of j mod 2^D (lines 52, 74), with one batch mean per codebook (line 120);
  * lfq_closed_form: the same loss without the C * 2^D softmax, in the closed form the kernels compute: with q the
    factorised distribution of a slice, eps' = C eps and H'(p) = -sum p log max(p, eps'),
        w_e [mean_r H'(q_r) + w_div mean_c H'(mean_n q_(n,c)) + (1 + w_div) log C] + w_c mse;
  * tokenizer_tokenize / tokenizer_forward: VideoTokenizer with this quantiser.
oracle/make_golden_lfq_multi.py checks every function here against the unmodified reference.
"""
import math

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import genie_oracle as O

EPS = 1e-6


def lfq_codebook(d: int, c: int) -> Tensor:
    """quantization.py:52,74-75 — c * 2^d rows; row j = bits of j & (2^d - 1), MSB first, mapped to {-1,+1}."""
    codes = torch.arange((2 ** d) * c)[:, None] & O.lfq_bit_mask(d)
    return 2 * (codes != 0).float() - 1


def lfq(x: Tensor, d: int, c: int, training: bool, beta: float = 100., transpose: bool = False,
        commit_weight: float = .25, entropy_weight: float = .1, diversity_weight: float = 1.,
        proj_inp=None, proj_out=None):
    """LookupFreeQuantization.forward with num_codebook = c — quantization.py:77-133, literally.
    Returns ((out, idxs), loss-or-None); ``idxs`` has shape (..., c) before the reference's ``.squeeze()``."""
    inp = x.movedim(1, -1) if transpose else x                     # 'b d ... -> b ... d'      (85)
    lead = inp.shape[1:-1]
    inp = inp.reshape(inp.shape[0], -1, inp.shape[-1])             # pack 'b * d'              (86)
    if proj_inp is not None:
        inp = F.linear(inp, proj_inp[0], proj_inp[1])              #                           (88)
    inp = inp.unflatten(-1, (c, d))                                # 'b n (c d) -> b n c d'    (91)
    quant = inp.sign()                                             #                           (97)
    idxs = ((inp > 0).int() * O.lfq_bit_mask(d).to(inp.device).int()).sum(-1)     # (b, n, c)   (98)
    code = (inp + (quant - inp).detach()) if training else quant   # STE                       (101)
    code = code.flatten(2)                                         # 'b n c d -> b n (c d)'    (102)
    out = code if proj_out is None else F.linear(code, proj_out[0], proj_out[1])   #           (105)
    out = out.reshape(out.shape[0], *lead, out.shape[-1])
    out = out.movedim(-1, 1) if transpose else out
    idxs = idxs.reshape(idxs.shape[0], *lead, c).squeeze()         #                           (110)
    if not training:
        return (out, idxs), None
    logits = 2 * torch.einsum('bncd,jd->bncj', inp, lfq_codebook(d, c).to(inp))    #           (116)
    prob = (logits * beta).softmax(dim=-1)                         #                           (117)
    prob = prob.flatten(0, 1)                                      # (b n) c j                 (118)
    avg_prob = prob.mean(dim=0)                                    # c j                       (120)
    inp_ent = O.lfq_entropy(prob).mean()
    avg_ent = O.lfq_entropy(avg_prob).mean()
    entropy_loss = inp_ent + diversity_weight * avg_ent            #                           (125)
    commit = F.mse_loss(inp, quant.detach())                       #                           (128)
    return (out, idxs), entropy_loss * entropy_weight + commit * commit_weight     #           (131)


def row_probs(rows: Tensor, beta: float = 100.) -> Tensor:
    """q [R, 2^D]: the factorised code distribution of each D-wide row, prod_d sigmoid(+-4 beta x_d), MSB first."""
    t = 4 * beta * rows
    sp, sm = torch.sigmoid(t), torch.sigmoid(-t)
    q = torch.ones(rows.shape[0], 1, dtype=rows.dtype, device=rows.device)
    for i in range(rows.shape[1]):
        q = torch.stack((q * sm[:, i, None], q * sp[:, i, None]), -1).flatten(1)
    return q


def lfq_closed_form(x2d: Tensor, d: int, c: int, beta: float = 100., commit_weight: float = .25,
                    entropy_weight: float = .1, diversity_weight: float = 1.) -> Tensor:
    """The training loss of lfq() on x2d [N, c*d] (no projection) without the c * 2^d softmax: each code's c copies
    carry q/c, so H(p) = H_{c eps}(q) + log c per row and per codebook mean."""
    n = x2d.shape[0]
    rows = x2d.reshape(n * c, d)
    q = row_probs(rows, beta)
    ent = lambda p: -(p * p.clamp(min=c * EPS).log()).sum(-1)
    avg = q.reshape(n, c, -1).mean(0)                              # one batch mean per codebook
    commit = ((rows - rows.sign()) ** 2).mean()
    return (entropy_weight * (ent(q).mean() + diversity_weight * ent(avg).mean() + (1 + diversity_weight) * math.log(c))
            + commit_weight * commit)


def _proj(sd, which):
    k = f'quant.{which}.weight'
    return (sd[k], sd.get(f'quant.{which}.bias')) if k in sd else None


def tokenizer_tokenize(sd, enc_bp, video: Tensor, d_codebook: int, n_codebook: int, beta: float = 100.):
    """VideoTokenizer.tokenize — tokenizer.py:332-350 with n_codebook codebooks."""
    enc = O.tokenizer_encode(sd, enc_bp, video)
    (q, idxs), _ = lfq(enc, d_codebook, n_codebook, training=False, beta=beta, transpose=True,
                       proj_inp=_proj(sd, 'proj_inp'), proj_out=_proj(sd, 'proj_out'))
    return q, idxs


def tokenizer_forward(sd, enc_bp, dec_bp, video: Tensor, d_codebook: int, n_codebook: int, beta: float = 100.,
                      quant_loss_weight: float = 1.):
    """VideoTokenizer.forward in training mode (GAN / perceptual terms at zero weight) with n_codebook codebooks.
    Returns (loss, (rec_loss, quant_loss), rec_video, idxs)."""
    enc = O.tokenizer_encode(sd, enc_bp, video)
    (q, idxs), q_loss = lfq(enc, d_codebook, n_codebook, training=True, beta=beta, transpose=True,
                            proj_inp=_proj(sd, 'proj_inp'), proj_out=_proj(sd, 'proj_out'))
    rec = O.tokenizer_decode(sd, dec_bp, q)
    rec_loss = F.mse_loss(rec, video)
    return rec_loss + q_loss * quant_loss_weight, (rec_loss, q_loss), rec, idxs
