"""Lookup-Free Quantization — mirrors genie/module/quantization.py:32-133 (same constructor, buffers,
return structure `((out, idxs), loss | None)`), computed by the fused LFQ kernels (csrc/lfq.cu) that never
materialise the (tokens x 2^D) softmax. With num_codebook = C > 1 every token's C*D inputs are C independent D-bit
codes, and the loss is the reference's over its C*2^D-row codebook (each code repeated C times), in closed form."""
from __future__ import annotations

from typing import Tuple

import torch
import torch.nn as nn
from torch import Tensor

from .. import ops
from ..utils import default


class LookupFreeQuantization(nn.Module):
    def __init__(self, codebook_dim: int, num_codebook: int = 1, input_dim: int | None = None, use_bias: bool = True,
                 frac_sample: float = 1., commit_weight: float = 0.25, entropy_weight: float = 0.1,
                 diversity_weight: float = 1.) -> None:
        super().__init__()
        if num_codebook < 1:
            raise ValueError(f'num_codebook must be >= 1, got {num_codebook}')
        codebook_size = (2 ** codebook_dim) * num_codebook
        input_dim = default(input_dim, codebook_size)
        project = input_dim != codebook_dim * num_codebook
        self.proj_inp = nn.Linear(input_dim, codebook_dim * num_codebook, bias=use_bias) if project else nn.Identity()
        self.proj_out = nn.Linear(codebook_dim * num_codebook, input_dim, bias=use_bias) if project else nn.Identity()
        self.frac_sample = frac_sample
        self.codebook_dim = codebook_dim
        self.num_codebooks = num_codebook
        self.codebook_size = codebook_size
        self.commit_weight = commit_weight
        self.entropy_weight = entropy_weight
        self.diversity_weight = diversity_weight
        self.register_buffer('bit_mask', 2 ** torch.arange(codebook_dim - 1, -1, -1))

    @property
    def codebook(self) -> Tensor:
        """The reference's codebook (quantization.py:74-75): codebook_size = C * 2^D rows, row j the sign code of j mod
        2^D, so each code appears C times. Built on demand — the kernels never need it."""
        codes = torch.arange(self.codebook_size, device=self.bit_mask.device)[:, None] & self.bit_mask
        return 2 * (codes != 0).float() - 1

    def codes_from_indices(self, idxs: Tensor) -> Tensor:
        """Token ids (b, t, h, w) -> the tensor `decode` expects, (b, C, t, h, w): bits (MSB first, `bit_mask`) -> +-1
        codes -> proj_out. The inverse of the packing on quantization.py:98 followed by line 105; needed by the
        inference roll-out (genie/genie.py:103 hands raw ids to decode, which cannot work). With num_codebook > 1 the
        ids are (b, t, h, w, num_codebook), one per codebook, as `forward` returns them before its `.squeeze()`."""
        bits = (idxs[..., None] & self.bit_mask.to(idxs.device)) != 0
        codes = bits.to(torch.float32) * 2 - 1
        if self.num_codebooks > 1:
            if idxs.shape[-1] != self.num_codebooks:
                raise ValueError(f'codes_from_indices: expected ids of shape (..., {self.num_codebooks}), '
                                 f'got {tuple(idxs.shape)}')
            codes = codes.flatten(-2)                                   # 'c d -> (c d)', quantization.py:102
        out = self.proj_out(codes)
        return out.movedim(-1, 1).contiguous()

    def forward(self, inp: Tensor, beta: float = 100., transpose: bool = False
                ) -> Tuple[Tuple[Tensor, Tensor], Tensor | None]:
        # 'b d ... -> b ... d' is free for internal-format (NDHWC) tensors
        x = inp.movedim(1, -1) if transpose else inp
        lead = x.shape[:-1]
        x = x.reshape(-1, x.shape[-1])
        if x.dtype != torch.float32:
            x = x.float()
        x = self.proj_inp(x)
        out, idxs, loss = ops.lfq(x, self.codebook_dim, beta, self.training, self.commit_weight,
                                  self.entropy_weight, self.diversity_weight, self.num_codebooks)
        out = self.proj_out(out)
        out = out.reshape(*lead, out.shape[-1])
        out = out.movedim(-1, 1) if transpose else out
        idxs = idxs.reshape(*lead, self.num_codebooks).squeeze()   # reference keeps .squeeze() (line 110)
        if not self.training:
            return (out, idxs), None
        return (out, idxs), loss
