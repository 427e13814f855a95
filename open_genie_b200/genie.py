"""Genie — the composed training module (genie/genie.py:18-181), RE-SPECIFIED per SURVEY.md §8 a15.

The reference constructor cannot run at HEAD (it reads undefined attributes such as self.enc_desc / TEST_DESC,
genie.py:37-58) and compute_loss forwards the (quant, idxs) tuple of tokenize() to the dynamics model
(genie.py:109). The intended data flow is kept, with explicit constructor arguments:

    with no_grad: _, tokens = tokenizer.tokenize(video)          # frozen tokenizer
    act_id, act_loss, (rec, q) = latent_action(video)
    dyn_loss = dynamics_model.compute_loss(tokens, act_id[, mask])
    loss = act_loss + dyn_loss                                    # logged as train/act_loss, train/dyn_loss, ...
"""
from __future__ import annotations

from typing import Callable, Iterable

import torch
from torch import Tensor
from torch.optim import Optimizer

from .action import LatentAction
from .dynamics import DynamicsModel
from .lightning_compat import LightningModule
from .optim import FusedAdamW
from .tokenizer import VideoTokenizer
from .utils import Blueprint

OptimizerCallable = Callable[[Iterable], Optimizer]


class Genie(LightningModule):
    def __init__(self, tokenizer: VideoTokenizer, latent_action: LatentAction | dict, dynamics_model: DynamicsModel | dict,
                 optimizer: OptimizerCallable = FusedAdamW, img_prompt: Tensor | None = None):
        super().__init__()
        if tokenizer.quant.num_codebooks != 1:
            raise NotImplementedError(f'Genie needs a tokenizer with n_codebook = 1 (got '
                                      f'{tokenizer.quant.num_codebooks}): DynamicsModel takes one token id per '
                                      f'position, (B, T, H, W)')
        self.tokenizer = tokenizer.requires_grad_(False)          # pre-trained, frozen (find_unused_parameters=False)
        self.latent_action = latent_action if isinstance(latent_action, LatentAction) else LatentAction(**latent_action)
        self.dynamics_model = (dynamics_model if isinstance(dynamics_model, DynamicsModel)
                               else DynamicsModel(**dynamics_model))
        self.optimizer = optimizer
        self.img_prompt = img_prompt
        self.save_hyperparameters(ignore=['tokenizer', 'latent_action', 'dynamics_model'])

    @torch.no_grad()
    def forward(self, prompt: Tensor, actions: Tensor, num_frames: int | None = None, steps_per_frame: int = 25) -> Tensor:
        """Inference: roll a video out of an image / clip prompt and a sequence of latent actions — the intent of
        genie/genie.py:65-105, RE-SPECIFIED where HEAD cannot run: `tokenize` returns `(quant, idxs)` (the reference
        forwards the tuple, line 89); each `generate` call already returns history + new frame (dynamics.py:163), so the
        `torch.stack` of line 100 is dropped; frame k of the roll-out is conditioned on one action per existing frame,
        `actions[:, :t]` (the reference slices with the loop index, which is empty on the first iteration); token ids
        are turned back into codes (LookupFreeQuantization.codes_from_indices) before `decode` (line 103 passes ids).
        prompt: (b,h,w) | (b,c,h,w) | (b,c,t,h,w); actions: (b, >= t0 + num_frames - 1) int64. Returns NCDHW fp32."""
        num_frames = actions.shape[1] if num_frames is None else num_frames
        match prompt.dim():
            case 3:
                prompt = prompt[:, None, None]
            case 4:
                prompt = prompt[:, :, None]
            case 5:
                pass
            case _:
                raise ValueError('Prompt must have 3, 4 or 5 dimensions')
        if actions.dim() == 1:
            actions = actions[None].expand(prompt.shape[0], -1)
        _, tokens = self.tokenizer.tokenize(prompt)
        if tokens.dim() == 3:                                   # the reference's .squeeze() drops singleton dims
            tokens = tokens.reshape(prompt.shape[0], -1, *tokens.shape[-2:])
        for _ in range(num_frames):
            t = tokens.shape[1]
            if actions.shape[1] < t:
                raise ValueError(f'need one action per generated transition: {actions.shape[1]} actions for {t} frames')
            tokens = self.dynamics_model.generate(tokens, actions[:, :t], steps=steps_per_frame)
        quant = self.tokenizer.quant.codes_from_indices(tokens)
        return self.tokenizer.decode(quant)

    def compute_loss(self, video: Tensor, mask: Tensor | None = None):
        with torch.no_grad():
            _, tokens = self.tokenizer.tokenize(video)
        act_id, act_loss, (act_rec_loss, act_q_loss) = self.latent_action(video)
        dyn_loss = self.dynamics_model.compute_loss(tokens, act_id, mask=mask)
        loss = act_loss + dyn_loss
        return loss, (('act_loss', act_loss), ('dyn_loss', dyn_loss), ('act_rec_loss', act_rec_loss),
                      ('act_q_loss', act_q_loss))

    def training_step(self, batch: Tensor, batch_idx: int) -> Tensor:
        loss, aux_losses = self.compute_loss(batch)
        self.log_dict({**{'train_loss': loss}, **{f'train/{k}': v for k, v in aux_losses}}, logger=True, on_step=True,
                      sync_dist=True)
        return loss

    def validation_step(self, batch: Tensor, batch_idx: int) -> Tensor:
        loss, aux_losses = self.compute_loss(batch)
        self.log_dict({**{'val_loss': loss}, **{f'val/{k}': v for k, v in aux_losses}}, logger=True, on_step=True,
                      sync_dist=True)
        return loss

    def on_validation_end(self) -> None:
        """genie/genie.py:155-174: roll out a sample video from `img_prompt` (or noise) and random actions and hand it
        to the logger when one is attached (`self.logger.experiment.add_video`)."""
        num_frames = 16
        dev = next(self.dynamics_model.parameters()).device
        prompt = self.img_prompt if self.img_prompt is not None else torch.randn(1, 3, 64, 64)
        actions = torch.randint(0, self.dynamics_model.act_vocab, size=(1, num_frames), device=dev)
        video = self(prompt.to(dev), actions, num_frames=num_frames, steps_per_frame=25)
        self.last_generated_video = video
        logger = getattr(self, 'logger', None)
        if logger is not None and hasattr(getattr(logger, 'experiment', None), 'add_video'):
            logger.experiment.add_video('Generated Video #1', video, global_step=getattr(self, 'global_step', 0))

    def configure_optimizers(self) -> Optimizer:
        return self.optimizer([p for p in self.parameters() if p.requires_grad])
