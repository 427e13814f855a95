"""DynamicsModel — mirrors genie/dynamics.py:14-194 (MaskGIT dynamics over space-time transformer blocks) on the
CUDA kernels: fused token+action embedding, SpaceTimeAttention blocks, the vocabulary head on the wgmma GEMM
kernel, a fused masked cross entropy. Same constructor, forward / compute_loss / generate / get_schedule
signatures, return values and state_dict keys (tok_emb.weight, act_emb.0.weight, head.{weight,bias},
dec_layers.N.*)."""
from __future__ import annotations

from math import pi, prod
from typing import Literal

import torch
import torch.nn as nn
from torch import Tensor

from . import ops
from .module import parse_blueprint
from .module.linear import LinearRows
from .utils import Blueprint, default


class DynamicsModel(nn.Module):
    def __init__(self, desc: Blueprint, tok_vocab: int, act_vocab: int, embed_dim: int) -> None:
        super().__init__()
        self.dec_layers, self.ext_kw = parse_blueprint(desc)
        self.head = LinearRows(embed_dim, tok_vocab)
        self.tok_emb = nn.Embedding(tok_vocab, embed_dim)
        self.act_emb = nn.Sequential(nn.Embedding(act_vocab, embed_dim), nn.Identity())
        self.tok_vocab, self.act_vocab, self.embed_dim = tok_vocab, act_vocab, embed_dim

    def _logits(self, tokens: Tensor, act_id: Tensor) -> Tensor:
        x = ops.embed_add(tokens, act_id, self.tok_emb.weight, self.act_emb[0].weight)      # (B,T,H,W,C) bf16
        for dec in self.dec_layers:
            x = dec(x)
        return self.head(x)                                                                  # (B,T,H,W,V) bf16

    def forward(self, tokens: Tensor, act_id: Tensor):
        """genie/dynamics.py:44-64: returns (logits (B,T,H,W,V), logits[:, -1])."""
        logits = self._logits(tokens, act_id).float()
        return logits, logits[:, -1]

    def compute_loss(self, tokens: Tensor, act_id: Tensor, mask: Tensor | None = None, fill: float = 0.) -> Tensor:
        """genie/dynamics.py:66-99 — including its quirk that the target is read from the ALREADY-masked tokens."""
        b, t, h, w = tokens.shape
        if mask is None:
            rate = torch.empty(1).uniform_(0.5, 1).item()
            mask = torch.distributions.Bernoulli(rate).sample((b, t, h, w)).bool()
        mask = mask.to(tokens.device)
        tokens = torch.masked_fill(tokens, mask, fill)
        logits = self._logits(tokens, act_id.detach())
        return ops.masked_cross_entropy(logits.reshape(-1, logits.shape[-1]), tokens, mask)

    @torch.no_grad()
    def generate(self, tokens: Tensor, act_id: Tensor, steps: int = 10,
                 which: Literal['linear', 'cosine', 'arccos'] = 'linear', temp: float = 1., topk: int = 50,
                 masked_tok: int = 0, uniforms: Tensor | None = None) -> Tensor:
        """MaskGIT iterative sampling of the next frame — genie/dynamics.py:101-165, as written there.

        The reference packs the transformer input `[tokens, code]` once BEFORE its loop (lines 128-134) and never
        refreshes it, so every iteration evaluates the model on the same input and only the multinomial draws differ
        (`topk` is accepted and unused there, too). Here the transformer therefore runs ONCE, and all iterations —
        softmax, draw, confidence, -inf on fixed positions, top-k, scatter — run in one fused launch
        (ops.maskgit_sample). `uniforms` (steps, b*h*w) optionally injects the draws (parity tests); by default they
        come from torch's CUDA generator. Returns pred_tok (b, t+1, h, w)."""
        b, t, h, w = tokens.shape
        schedule = self.get_schedule(steps, shape=(h, w), which=which)
        code0 = torch.full((b, 1, h, w), masked_tok, device=tokens.device, dtype=tokens.dtype)
        mock = torch.zeros(b, 1, dtype=act_id.dtype, device=tokens.device)
        tok_id = torch.cat([tokens, code0], dim=1)
        act_all = torch.cat([act_id.to(tokens.device), mock], dim=1)
        logits_last = self._logits(tok_id, act_all)[:, -1]                        # (b, h, w, V) bf16
        if uniforms is None:
            uniforms = torch.rand((steps, b * h * w), device=tokens.device)
        code, mask = ops.maskgit_sample(logits_last, uniforms, schedule, temp=temp, masked_tok=masked_tok)
        left = int(mask.sum())
        assert left == 0, f'Not all tokens were predicted. {left} tokens left.'
        return torch.cat([tokens, code[:, None].to(tokens.dtype)], dim=1)

    def get_schedule(self, steps: int, shape: tuple[int, int],
                     which: Literal['linear', 'cosine', 'arccos'] = 'linear') -> Tensor:
        """genie/dynamics.py:167-194."""
        n = prod(shape)
        t = torch.linspace(1, 0, steps)
        match which:
            case 'linear':
                s = 1 - t
            case 'cosine':
                s = torch.cos(t * pi * .5)
            case 'arccos':
                s = torch.acos(t) / (pi * .5)
            case _:
                raise ValueError(f'Unknown schedule type: {which}')
        schedule = (s / s.sum()) * n
        schedule = schedule.round().int().clamp(min=1)
        schedule[-1] += n - schedule.sum()
        return schedule
