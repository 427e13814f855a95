"""Minimal stand-in for the `lightning` package (not installed in this image) so the UNMODIFIED
reference checkout can be imported by oracle/make_golden.py. Test infrastructure only."""
import torch.nn as nn


class LightningModule(nn.Module):
    def save_hyperparameters(self, *a, **k):
        pass

    def log_dict(self, *a, **k):
        pass

    def log(self, *a, **k):
        pass


class LightningDataModule:
    def __init__(self, *a, **k):
        pass
