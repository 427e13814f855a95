"""VideoTokenizer — the reference's Lightning surface (genie/tokenizer.py:225-442) on the H100 hot path.

Same constructor signature, blueprints, method names, return tuples, logged metric keys and state_dict
keys, including the GAN (frame critic, hinge losses) and perceptual (VGG16 feature distance) terms of
genie/module/loss.py — see open_genie_b200/module/loss.py for the two facts that matter there (the perceptual
term carries no gradient in the reference; VGG16 weights cannot be downloaded offline)."""
from __future__ import annotations

from typing import Any, Callable, Dict, Iterable, Tuple

import torch
import torch.nn as nn
from torch import Tensor
from torch.optim import Optimizer

from . import ops
from .lightning_compat import LightningModule
from .module import parse_blueprint
from .module.quantization import LookupFreeQuantization
from .module.video import CausalConv3d
from .optim import FusedAdamW
from .utils import Blueprint, default, exists

OptimizerCallable = Callable[[Iterable], Optimizer]

# Blueprints: identical content to genie/tokenizer.py:24-205 (they are configuration, i.e. the API).
MAGVIT2_ENC_DESC = (
    ('causal-conv3d', {'in_channels': 3, 'out_channels': 128, 'kernel_size': 3}),
    ('video-residual', {'n_rep': 4, 'in_channels': 128}),
    ('spacetime_downsample', {'in_channels': 128, 'out_channels': 128, 'kernel_size': 3, 'time_factor': 1,
                              'space_factor': 2}),
    ('video-residual', {'in_channels': 128, 'out_channels': 256}),
    ('video-residual', {'n_rep': 3, 'in_channels': 256}),
    ('spacetime_downsample', {'in_channels': 256, 'out_channels': 256, 'kernel_size': 3, 'time_factor': 2,
                              'space_factor': 2}),
    ('video-residual', {'n_rep': 4, 'in_channels': 256}),
    ('spacetime_downsample', {'in_channels': 256, 'out_channels': 256, 'kernel_size': 3, 'time_factor': 2,
                              'space_factor': 2}),
    ('video-residual', {'in_channels': 256, 'out_channels': 512}),
    ('video-residual', {'n_rep': 7, 'in_channels': 512}),
    ('group_norm', {'num_groups': 8, 'num_channels': 512}),
    ('silu', {}),
    ('causal-conv3d', {'in_channels': 512, 'out_channels': 18, 'kernel_size': 1}),
)

MAGVIT2_DEC_DESC = (
    ('causal-conv3d', {'in_channels': 18, 'out_channels': 512, 'kernel_size': 3}),
    ('video-residual', {'n_rep': 4, 'in_channels': 512}),
    ('adaptive_group_norm', {'dim_cond': 18, 'num_groups': 8, 'num_channels': 512, 'has_ext': True}),
    ('video-residual', {'n_rep': 4, 'in_channels': 512}),
    ('depth2spacetime_upsample', {'in_channels': 512, 'kernel_size': 3, 'time_factor': 2, 'space_factor': 2}),
    ('adaptive_group_norm', {'dim_cond': 18, 'num_groups': 8, 'num_channels': 512, 'has_ext': True}),
    ('video-residual', {'in_channels': 512, 'out_channels': 256}),
    ('video-residual', {'n_rep': 3, 'in_channels': 256}),
    ('depth2spacetime_upsample', {'in_channels': 256, 'kernel_size': 3, 'time_factor': 2, 'space_factor': 2}),
    ('adaptive_group_norm', {'dim_cond': 18, 'num_groups': 8, 'num_channels': 256, 'has_ext': True}),
    ('video-residual', {'n_rep': 4, 'in_channels': 256}),
    ('depth2spacetime_upsample', {'in_channels': 256, 'kernel_size': 3, 'time_factor': 1, 'space_factor': 2}),
    ('adaptive_group_norm', {'dim_cond': 18, 'num_groups': 8, 'num_channels': 256, 'has_ext': True}),
    ('video-residual', {'in_channels': 256, 'out_channels': 128}),
    ('video-residual', {'n_rep': 3, 'in_channels': 128}),
    ('group_norm', {'num_groups': 8, 'num_channels': 128}),
    ('silu', {}),
    ('causal-conv3d', {'in_channels': 128, 'out_channels': 3, 'kernel_size': 3}),
)

REPR_TOK_ENC = (
    ('spacetime_downsample', {'in_channels': 3, 'kernel_size': 3, 'out_channels': 512, 'time_factor': 1,
                              'space_factor': 4}),
    ('space-time_attn', {'n_rep': 8, 'n_head': 8, 'd_head': 64, 'transpose': True}),
)

REPR_TOK_DEC = (
    ('space-time_attn', {'n_rep': 8, 'n_head': 8, 'd_head': 64, 'transpose': True}),
    ('depth2spacetime_upsample', {'in_channels': 512, 'kernel_size': 3, 'out_channels': 3, 'time_factor': 1,
                                  'space_factor': 4}),
)


def get_enc(name: str) -> Blueprint:
    match name:
        case 'magvit2':
            return MAGVIT2_ENC_DESC
        case 'repr_tok':
            return REPR_TOK_ENC
        case _:
            raise ValueError(f'Unknown encoder: {name}')


def get_dec(name: str) -> Blueprint:
    match name:
        case 'magvit2':
            return MAGVIT2_DEC_DESC
        case 'repr_tok':
            return REPR_TOK_DEC
        case _:
            raise ValueError(f'Unknown decoder: {name}')


class VideoTokenizer(LightningModule):
    """MagViT-2 style video tokenizer: encode -> lookup-free quantise -> decode."""

    def __init__(
        self,
        enc_desc: Blueprint,
        dec_desc: Blueprint,
        disc_kwargs: Dict[str, Any] = {},
        d_codebook: int = 18,
        n_codebook: int = 1,
        lfq_bias: bool = True,
        lfq_frac_sample: float = 1.,
        lfq_commit_weight: float = 0.25,
        lfq_entropy_weight: float = 0.1,
        lfq_diversity_weight: float = 1.,
        optimizer: OptimizerCallable = FusedAdamW,
        perceptual_model: str = 'vgg16',
        perc_feat_layers: str | Iterable[str] = ('features.6', 'features.13', 'features.18', 'features.25'),
        gan_discriminate: str = 'frames',
        gan_frames_per_batch: int = 4,
        gan_loss_weight: float = 1.,
        perc_loss_weight: float = 1.,
        quant_loss_weight: float = 1.,
    ) -> None:
        super().__init__()
        self.optimizer = optimizer
        self.enc_layers, self.enc_ext = parse_blueprint(enc_desc)
        self.dec_layers, self.dec_ext = parse_blueprint(dec_desc)
        last_enc_dim = [m.out_channels for m in self.enc_layers.modules() if hasattr(m, 'out_channels')][-1]
        first_dec_dim = self.dec_layers[0].in_channels
        assert last_enc_dim == first_dec_dim, 'Inconsistent encoder/decoder dimensions'
        self.quant = LookupFreeQuantization(
            codebook_dim=d_codebook, num_codebook=n_codebook, input_dim=last_enc_dim, use_bias=lfq_bias,
            frac_sample=lfq_frac_sample, commit_weight=lfq_commit_weight, entropy_weight=lfq_entropy_weight,
            diversity_weight=lfq_diversity_weight)
        # auxiliary objectives (genie/tokenizer.py:288-299); a disabled term is identically zero here (the reference
        # calls nn.Identity()(rec, video, train_gen=True) in that case and raises)
        from .module.loss import GANLoss, PerceptualLoss
        self.perc_crit = PerceptualLoss(model_name=perceptual_model, feat_layers=perc_feat_layers,
                                        num_frames=gan_frames_per_batch) if perc_loss_weight > 0 else nn.Identity()
        self.gan_crit = GANLoss(discriminate=gan_discriminate, num_frames=gan_frames_per_batch,
                                **disc_kwargs) if gan_loss_weight > 0 else nn.Identity()
        self.gan_loss_weight = gan_loss_weight
        self.perc_loss_weight = perc_loss_weight
        self.quant_loss_weight = quant_loss_weight
        # the tensors that feed a loss stay fp32: encoder head -> LFQ, decoder tail -> mse
        for layers in (self.enc_layers, self.dec_layers):
            if len(layers) and isinstance(layers[-1], CausalConv3d):
                layers[-1].out_f32 = True
        self.save_hyperparameters()

    # ---- reference surface ------------------------------------------------------------------
    def encode(self, video: Tensor, cond: Tensor | None = None) -> Tensor:
        """genie/tokenizer.py:307-317. Returns the latent in internal format (use ops.to_reference for NCDHW)."""
        enc_video = video
        for layer, has_ext in zip(self.enc_layers, self.enc_ext):
            enc_video = layer(enc_video, cond) if has_ext else layer(enc_video)
        return enc_video

    def _decode_internal(self, quant: Tensor, cond: Tensor | None = None) -> Tensor:
        cond = default(cond, quant)
        rec_video = quant
        for layer, has_ext in zip(self.dec_layers, self.dec_ext):
            rec_video = layer(rec_video, cond) if has_ext else layer(rec_video)
        return rec_video

    def decode(self, quant: Tensor, cond: Tensor | None = None) -> Tensor:
        """genie/tokenizer.py:319-330; returns NCDHW fp32 like the reference."""
        return ops.to_reference(self._decode_internal(quant, cond))

    @torch.no_grad()
    def tokenize(self, video: Tensor, beta: float = 100., transpose: bool = True) -> Tuple[Tensor, Tensor]:
        """genie/tokenizer.py:332-350 (including its quirk of leaving the module in train mode)."""
        self.eval()
        enc_video = self.encode(video)
        (quant_video, idxs), _ = self.quant(enc_video, beta=beta, transpose=transpose)
        self.train()
        return ops.to_reference(quant_video) if quant_video.dim() == 5 else quant_video, idxs

    def forward(self, video: Tensor, beta: float = 100., transpose: bool = True
                ) -> Tuple[Tensor, Tuple[Tensor, ...]]:
        """genie/tokenizer.py:352-387 with the GAN / perceptual terms identically zero."""
        enc_video = self.encode(video)
        (quant_video, idxs), quant_loss = self.quant(enc_video, beta=beta, transpose=transpose)
        rec_video = self._decode_internal(quant_video)
        rec_loss = ops.mse_loss(rec_video, video)
        gen_loss = dis_loss = perc_loss = 0.
        if self.gan_loss_weight > 0:           # hinge GAN on randomly picked frames (tokenizer.py:367-368)
            gen_loss = self.gan_crit(rec_video, video, train_gen=True)
            dis_loss = self.gan_crit(rec_video, video, train_gen=False)
        if self.perc_loss_weight > 0:          # VGG16 feature distance (tokenizer.py:371); carries no gradient
            perc_loss = self.perc_crit(rec_video, video)
        # the reference's operator precedence (lines 375-379): in eval mode (quant_loss None) the loss is 0
        loss = (rec_loss + gen_loss * self.gan_loss_weight + dis_loss * self.gan_loss_weight
                + perc_loss * self.perc_loss_weight + quant_loss * self.quant_loss_weight) if exists(quant_loss) else 0
        return loss, (
            rec_loss,
            gen_loss if self.gan_loss_weight > 0 else 0,
            dis_loss if self.gan_loss_weight > 0 else 0,
            perc_loss if self.perc_loss_weight > 0 else 0,
            quant_loss if exists(quant_loss) and self.quant_loss_weight > 0 else 0,
        )

    # ---- Lightning hooks ---------------------------------------------------------------------
    def training_step(self, batch: Tensor, batch_idx: int) -> Tensor:
        loss, aux_losses = self(batch)
        self.log_dict({'train_loss': loss, 'train_rec_loss': aux_losses[0], 'train_gen_loss': aux_losses[1],
                       'train_dis_loss': aux_losses[2], 'train_perc_loss': aux_losses[3],
                       'train_quant_loss': aux_losses[4]}, logger=True, on_step=True, sync_dist=True)
        return loss

    def validation_step(self, batch: Tensor, batch_idx: int) -> Tensor:
        loss, aux_losses = self(batch)
        self.log_dict({'val_loss': loss, 'val_rec_loss': aux_losses[0], 'val_gen_loss': aux_losses[1],
                       'val_dis_loss': aux_losses[2], 'val_perc_loss': aux_losses[3],
                       'val_quant_loss': aux_losses[4]}, on_step=True, logger=True, sync_dist=True)
        return loss

    def on_validation_end(self) -> None:
        pass

    def configure_optimizers(self) -> Optimizer:
        return self.optimizer(self.parameters())
